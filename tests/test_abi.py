"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/gsql_gpu.h
declares, the Python binding table matches the header, and — with no GPU — the product path fails loudly instead
of falling back to the CPU."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "gsql_gpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gsql_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()
    from galaxysql_b200 import native as N
    lib = C.CDLL(N.SO_PATH)
    syms = header_symbols()
    assert len(syms) >= 40
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in gsql_gpu.h but not exported"
    assert sorted(N.ABI_SYMBOLS) == syms, "galaxysql_b200/native.py binding table is out of sync with the header"
    assert N.load().gsql_abi_version() == 2


def test_struct_layouts_match_header_sizes():
    """ctypes mirrors must have the C sizes (checked against a tiny C program compiled with gcc)."""
    import subprocess
    import tempfile
    from galaxysql_b200 import native as N
    prog = r'''
    #include <stdio.h>
    #include "gsql_gpu.h"
    int main(){ printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(gsql_col), sizeof(gsql_batch), sizeof(gsql_join_spec),
                       sizeof(gsql_join_info), sizeof(gsql_agg_call), sizeof(gsql_agg_spec), sizeof(gsql_xchg_spec),
                       sizeof(gsql_expr_ins), sizeof(gsql_expr), sizeof(gsql_scan_spec)); return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(prog)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        sizes = list(map(int, subprocess.check_output([os.path.join(d, "t")]).split()))
    got = [C.sizeof(x) for x in (N.Col, N.Batch, N.JoinSpec, N.JoinInfo, N.AggCall, N.AggSpec, N.XchgSpec, N.ExprIns, N.Expr, N.ScanSpec)]
    assert got == sizes


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    from galaxysql_b200 import api, native as N
    with pytest.raises(N.GsqlError):
        api.Context(0)


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "galaxysql_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                txt = open(os.path.join(dirpath, f), errors="replace").read()
                assert "import oracle" not in txt and "from oracle" not in txt and "oracle/" not in txt.replace("oracle/ is test", ""), f
