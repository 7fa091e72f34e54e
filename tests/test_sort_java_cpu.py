"""CPU checks of the Java side of ORDER BY / TOP-N (the image has no JDK, so javac cannot run; tests/test_jni_boundary.py
already checks that every GpuNative.sort* call site names a declared native with its arity, and that the shim defines
them):

* the operators and factories extend the reference types they replace, and every reference type they import is imported
  from the package the reference declares it in (paths cited in the class headers and in INTEGRATION.md);
* GpuTopNExecutorFactory keeps TopNExecutorFactory's topSize = skip + fetch, GpuTopNExec refuses topSize < 0 as
  SpilledTopNExec does, GpuSortExec asks for every row (limit -1) and passes DESC as isAsc() negated;
* GpuSupport.sortSupported refuses types without a GPU block form (DECIMAL, CHAR, ...), more keys than GSQL_MAX_KEYS and
  more columns than GSQL_MAX_COLS;
* INTEGRATION.md gives the visitMemSort / visitTopN patches as code."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")

FILES = {
    "GpuSortExec": "operator/GpuSortExec.java",
    "GpuTopNExec": "operator/GpuTopNExec.java",
    "GpuSortExecutorFactory": "mpp/operator/factory/GpuSortExecutorFactory.java",
    "GpuTopNExecutorFactory": "mpp/operator/factory/GpuTopNExecutorFactory.java",
    "GpuSupport": "operator/gpu/GpuSupport.java",
}

# reference types the new classes use -> the package the reference declares them in (checked against the reference's
# sources when this list was written; the reference is not readable from the tests at run time, so the list is static)
REFERENCE_TYPES = {
    "OrderByOption": "com.alibaba.polardbx.executor.utils",            # EX/utils/OrderByOption.java
    "ExecUtils": "com.alibaba.polardbx.executor.utils",                # EX/utils/ExecUtils.java (convertFrom)
    "MemSort": "com.alibaba.polardbx.optimizer.core.rel",              # OPT/core/rel/MemSort.java
    "TopN": "com.alibaba.polardbx.optimizer.core.rel",                 # OPT/core/rel/TopN.java
    "RuntimeStatHelper": "com.alibaba.polardbx.statistics",            # as SortExecutorFactory / TopNExecutorFactory import it
    "ParameterContext": "com.alibaba.polardbx.common.jdbc",
    "RelFieldCollation": "org.apache.calcite.rel",
    "ExecutionContext": "com.alibaba.polardbx.optimizer.context",
    "DataType": "com.alibaba.polardbx.optimizer.core.datatype",
}
CITED = {  # the reference file each new class names as the one it replaces
    "GpuSortExec": ["operator/SortExec.java", "operator/util/MemSortor.java"],
    "GpuTopNExec": ["operator/SpilledTopNExec.java"],
    "GpuSortExecutorFactory": ["mpp/operator/factory/SortExecutorFactory.java"],
    "GpuTopNExecutorFactory": ["mpp/operator/factory/TopNExecutorFactory.java"],
}


def _src(name):
    return open(os.path.join(PKG, FILES[name])).read()


def _code(name):
    s = re.sub(r"/\*.*?\*/", "", _src(name), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def _header_defines():
    h = open(os.path.join(ROOT, "include", "gsql_gpu.h")).read()
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(GSQL_\w+)\s+(\d+)", h)}


def test_operators_and_factories_extend_what_they_replace():
    assert re.search(r"class GpuSortExec extends AbstractExecutor implements ConsumerExecutor\b", _code("GpuSortExec"))
    assert re.search(r"class GpuTopNExec extends GpuSortExec\b", _code("GpuTopNExec"))
    for f in ("GpuSortExecutorFactory", "GpuTopNExecutorFactory"):
        assert re.search(r"class " + f + r" extends ExecutorFactory\b", _code(f))
    for name, cited in CITED.items():
        for c in cited:
            assert c in _src(name), f"{name} does not cite {c}"
        assert c.split("/")[-1] in open(os.path.join(ROOT, "INTEGRATION.md")).read()


def test_reference_imports_come_from_the_reference_packages():
    for name in FILES:
        code = _code(name)
        pkg = re.search(r"^package\s+([\w.]+);", code, flags=re.M).group(1)
        for simple, ref_pkg in REFERENCE_TYPES.items():
            if not re.search(r"\b" + simple + r"\b", re.sub(r"^import[^\n]*\n", "", code, flags=re.M)):
                continue
            imported = re.findall(r"^import\s+([\w.]+)\." + simple + r";", code, flags=re.M)
            assert imported == [ref_pkg] or (not imported and pkg == ref_pkg), f"{name}: {simple} must come from {ref_pkg}, got {imported}"
    assert "import static com.alibaba.polardbx.optimizer.core.planner.rule.util.CBOUtil.getRexParam;" in _code("GpuTopNExecutorFactory")


def test_top_size_arithmetic_and_limits():
    f = _code("GpuTopNExecutorFactory")
    assert re.search(r"static long topSize\(long skip, long fetch\)\s*\{\s*return skip \+ fetch;", f)
    assert "long fetch = -1, skip = 0;" in f and "new GpuTopNExec(dataTypeList, orderBys, topSize(skip, fetch), context)" in f
    t = _code("GpuTopNExec")
    assert re.search(r"if \(topSize < 0\)\s*\{\s*throw new IllegalArgumentException\(\"topN not support top size:\" \+ topSize\);", t)
    s = _code("GpuSortExec")
    assert "this(dataTypes, orderBys, -1, context);" in s
    assert "keyDesc[i] = orderBys.get(i).isAsc() ? 0 : 1;" in s and "keyCols[i] = orderBys.get(i).getIndex();" in s
    assert "GpuNative.sortCreate(ctx, codes, keyCols, keyDesc, limit)" in s


def test_sort_supported_refuses_what_the_gpu_does_not_order():
    h = _header_defines()
    g = _code("GpuSupport")
    m = re.search(r"MAX_SORT_KEYS = (\d+), MAX_SORT_COLS = (\d+);", g)
    assert m and (int(m.group(1)), int(m.group(2))) == (h["GSQL_MAX_KEYS"], h["GSQL_MAX_COLS"])
    body = g[g.index("public static boolean sortSupported"):]
    body = body[:body.index("public static boolean aggSupported")]
    assert "collations.size() > MAX_SORT_KEYS" in body and "inputTypes.size() > MAX_SORT_COLS" in body
    assert "GpuTypes.supported(inputTypes)" in body and "!enabled(context)" in body
    # GpuTypes.code has no DECIMAL / CHAR form: such a column makes supported() false
    types = re.sub(r"/\*.*?\*/", "", open(os.path.join(PKG, "operator/gpu/GpuTypes.java")).read(), flags=re.S)
    code_fn = types[types.index("public static int code("):types.index("public static boolean isPackedTime")]
    assert "Decimal" not in code_fn and "String" not in code_fn and "Varchar" not in code_fn


def test_integration_gives_the_planner_patches_as_code():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("### ORDER BY / TOP-N"):]
    sec = sec[:sec.index("\n## ")]
    blocks = re.findall(r"```java\n(.*?)```", sec, flags=re.S)
    assert blocks, "no Java patch in the ORDER BY section"
    code = "\n".join(blocks)
    assert "visitMemSort" in code and "visitTopN" in code
    assert "new GpuSortExecutorFactory(sort, memSortParallelism, columns)" in code
    assert "new GpuTopNExecutorFactory(topN, pipelineFragment.getParallelism(), columns)" in code
    assert code.count("GpuSupport.sortSupported(") == 2
