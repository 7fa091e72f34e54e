"""CPU checks of the Java side of the merge of sorted runs (the image has no JDK; tests/test_jni_boundary.py already
checks every GpuNative.merge* call site against the declared natives and the shim):

* GpuMergeSortExec extends AbstractExecutor like MergeSortExec, GpuLocalMergeSortExecutorFactory extends ExecutorFactory
  like LocalMergeSortExecutorFactory, and each reference type they import comes from the package the reference declares
  it in;
* the GPU limit is offset + fetch saturating (an overflow means every row), the pass-through rule is the reference's
  ignoreMergeSort, and limit <= 0 opens nothing;
* the factory extracts offset / fetch as LocalMergeSortExecutorFactory does and falls back to the stock MergeSortExec;
* GpuSupport.mergeSortSupported keeps sortSupported's bounds and adds GSQL_MAX_MERGE_INPUTS;
* INTEGRATION.md gives the planner patch as code."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")

FILES = {
    "GpuMergeSortExec": "operator/GpuMergeSortExec.java",
    "GpuLocalMergeSortExecutorFactory": "mpp/operator/factory/GpuLocalMergeSortExecutorFactory.java",
    "GpuSupport": "operator/gpu/GpuSupport.java",
}

# reference types the new classes use -> the package the reference declares them in (static: the reference is not
# readable from the tests at run time)
REFERENCE_TYPES = {
    "OrderByOption": "com.alibaba.polardbx.executor.utils",
    "ExecUtils": "com.alibaba.polardbx.executor.utils",
    "MergeSortExec": "com.alibaba.polardbx.executor.operator",
    "Executor": "com.alibaba.polardbx.executor.operator",
    "RuntimeStatHelper": "com.alibaba.polardbx.statistics",
    "ParameterContext": "com.alibaba.polardbx.common.jdbc",
    "RelFieldCollation": "org.apache.calcite.rel",
    "Sort": "org.apache.calcite.rel.core",
    "ExecutionContext": "com.alibaba.polardbx.optimizer.context",
    "DataType": "com.alibaba.polardbx.optimizer.core.datatype",
}
CITED = {
    "GpuMergeSortExec": ["operator/MergeSortExec.java"],
    "GpuLocalMergeSortExecutorFactory": ["mpp/operator/factory/LocalMergeSortExecutorFactory.java"],
}


def _src(name):
    return open(os.path.join(PKG, FILES[name])).read()


def _code(name):
    s = re.sub(r"/\*.*?\*/", "", _src(name), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def test_classes_extend_what_they_replace_and_cite_it():
    assert re.search(r"class GpuMergeSortExec extends AbstractExecutor\s*\{", _code("GpuMergeSortExec"))
    assert re.search(r"class GpuLocalMergeSortExecutorFactory extends ExecutorFactory\b", _code("GpuLocalMergeSortExecutorFactory"))
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    for name, cited in CITED.items():
        for c in cited:
            assert c in _src(name), f"{name} does not cite {c}"
            assert c in doc
    assert re.search(r"public GpuMergeSortExec\(List<Executor> inputs, List<OrderByOption> orderBys, long offset, long limit,\s*"
                     r"ExecutionContext context\)", _code("GpuMergeSortExec"))
    assert "public GpuLocalMergeSortExecutorFactory(Sort sort, ExecutorFactory executorFactory, int childParallelism)" in \
        _code("GpuLocalMergeSortExecutorFactory")


def test_reference_imports_come_from_the_reference_packages():
    for name in FILES:
        code = _code(name)
        pkg = re.search(r"^package\s+([\w.]+);", code, flags=re.M).group(1)
        body = re.sub(r"^import[^\n]*\n", "", code, flags=re.M)
        for simple, ref_pkg in REFERENCE_TYPES.items():
            if not re.search(r"\b" + simple + r"\b", body):
                continue
            imported = re.findall(r"^import\s+([\w.]+)\." + simple + r";", code, flags=re.M)
            assert imported == [ref_pkg] or (not imported and pkg == ref_pkg), f"{name}: {simple} must come from {ref_pkg}, got {imported}"
    assert "import static com.alibaba.polardbx.optimizer.core.planner.rule.util.CBOUtil.getRexParam;" in _code("GpuLocalMergeSortExecutorFactory")


def test_offset_plus_fetch_saturates():
    e = _code("GpuMergeSortExec")
    assert re.search(r"static long gpuLimit\(long offset, long limit\)\s*\{\s*return limit >= Long\.MAX_VALUE - offset \? -1 : offset \+ limit;", e)
    assert "this.gpuLimit = gpuLimit(offset, limit);" in e
    assert "GpuNative.mergeCreate(ctx, codes, keyCols, keyDesc, inputs.size(), gpuLimit)" in e
    assert "keyDesc[i] = orderBys.get(i).isAsc() ? 0 : 1;" in e and "keyCols[i] = orderBys.get(i).getIndex();" in e
    # an input stops being pulled once it delivered the merge's quota
    assert re.search(r"if \(gpuLimit >= 0 && pulled\[i\] >= gpuLimit\)\s*\{\s*drained\[i\] = true;", e)


def test_pass_through_and_limit_at_most_zero():
    e = _code("GpuMergeSortExec")
    assert "this.ignoreMergeSort = inputs.size() == 1 && offset == 0 && limit == Long.MAX_VALUE;" in e
    open_body = e[e.index("void doOpen()"):e.index("private void flush()")]
    assert re.search(r"if \(limit <= 0\)\s*\{\s*return;\s*\}", open_body)
    assert re.search(r"if \(!ignoreMergeSort\)\s*\{\s*ctx = GpuNative\.ctxCreate", open_body)  # pass-through: no GPU handle
    nxt = e[e.index("Chunk doNextChunk()"):e.index("void doClose()")]
    assert re.search(r"if \(fetched <= 0 \|\| finished\)\s*\{\s*return null;", nxt)
    assert re.search(r"if \(ignoreMergeSort\)\s*\{\s*return passThrough\(\);", nxt)
    close_body = e[e.index("void doClose()"):e.index("public List<DataType> getDataTypes()")]
    assert re.search(r"if \(limit <= 0\)\s*\{\s*return;\s*\}", close_body)
    assert "produceIsBlocked()" in e[e.index("private boolean pull()"):]  # a blocked input's future is reported


def test_factory_extracts_offset_and_fetch_as_the_reference_does():
    f = _code("GpuLocalMergeSortExecutorFactory")
    assert "long limit = Long.MAX_VALUE;" in f and "long offset = 0;" in f
    assert re.search(r"if \(sort\.fetch != null\)\s*\{\s*limit = getRexParam\(sort\.fetch, params\);\s*if \(sort\.offset != null\)\s*\{\s*"
                     r"offset = getRexParam\(sort\.offset, params\);", f)
    assert "GpuSupport.mergeSortSupported(inputs.get(0).getDataTypes(), sortList, childParallelism, context)" in f
    assert "new GpuMergeSortExec(inputs, orderBys, offset, limit, context)" in f
    assert "new MergeSortExec(inputs, orderBys, offset, limit, context)" in f


def test_merge_sort_supported_bounds():
    h = open(os.path.join(ROOT, "include", "gsql_gpu.h")).read()
    max_inputs = int(re.search(r"#define\s+GSQL_MAX_MERGE_INPUTS\s+(\d+)", h).group(1))
    g = _code("GpuSupport")
    assert int(re.search(r"MAX_MERGE_INPUTS = (\d+);", g).group(1)) == max_inputs
    body = g[g.index("public static boolean mergeSortSupported"):]
    body = body[:body.index("public static boolean aggSupported")]
    assert "childParallelism < 1 || childParallelism > MAX_MERGE_INPUTS" in body
    assert "return sortSupported(inputTypes, collations, context);" in body


def test_integration_gives_the_planner_patch_as_code():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("### Merge of sorted runs"):]
    sec = sec[:sec.index("\n## ")]
    code = "\n".join(re.findall(r"```java\n(.*?)```", sec, flags=re.S))
    assert "visitMergeSort" in code
    assert "new GpuLocalMergeSortExecutorFactory(mergeSort, childExecutorFactory, childFragment.getParallelism())" in code
    assert "new GpuLocalMergeSortExecutorFactory(sort, factory, pipelineFragment.getParallelism())" in code
