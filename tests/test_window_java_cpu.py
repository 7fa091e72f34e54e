"""CPU checks of the Java side of the window operator (the image has no JDK; tests/test_jni_boundary.py already checks every
GpuNative.window* call site against the declared natives and the shim):

* GpuNonFrameOverWindowExec extends the stock NonFrameOverWindowExec and keeps its constructor's arguments;
* GpuNonFrameOverWindowExecFactory extends OverWindowFramesExecFactory and defers to super unless
  GpuSupport.nonFrameWindowSupported holds;
* refusals are made at planner time (first call of the rank family, one group, no FILTER, at most 4 RANK columns, no
  DECIMAL);
* the natives are declared and implemented, and INTEGRATION.md gives the planner patch."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")


def _code(rel):
    s = re.sub(r"/\*.*?\*/", "", open(os.path.join(PKG, rel)).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def test_executor_extends_the_stock_class():
    e = _code("operator/GpuNonFrameOverWindowExec.java")
    assert re.search(r"class GpuNonFrameOverWindowExec extends NonFrameOverWindowExec\s*\{", e)
    assert re.search(r"public GpuNonFrameOverWindowExec\(Executor input, ExecutionContext context, GpuAggSpec spec, "
                     r"List<Integer> partitionIndexes,\s*boolean resetEachRow, List<DataType> dataTypes\)", e)
    assert "GpuNative.windowApply(window, in, out)" in e
    # chunks are batched to GPU_BATCH_ROWS before a call, and flushed when the input blocks or finishes
    assert "if (GpuNative.stagingRows(in) >= GpuHashAggExec.GPU_BATCH_ROWS)" in e
    assert re.search(r"if \(chunk == null\)\s*\{[^}]*flush\(\);", e)
    assert "blocks[i] = chunk.getBlock(i);" in e  # the input blocks pass through unchanged
    assert "inputFinished = input.produceIsFinished();" in e and "blocked = input.produceIsBlocked();" in e


def test_factory_falls_back_to_super():
    f = _code("mpp/operator/factory/GpuNonFrameOverWindowExecFactory.java")
    assert re.search(r"class GpuNonFrameOverWindowExecFactory extends OverWindowFramesExecFactory\b", f)
    assert "public GpuNonFrameOverWindowExecFactory(SortWindow overWindow, ExecutorFactory executorFactory)" in f
    body = f[f.index("public Executor createExecutor"):]
    # the decision comes from the plan before any child exists; each branch creates the child once
    assert re.search(r"if \(!GpuSupport\.nonFrameWindowSupported\(overWindow, context\)\)\s*\{\s*"
                     r"return super\.createExecutor\(context, index\);\s*\}\s*"
                     r"Executor input = getInputs\(\)\.get\(0\)\.createExecutor\(context, index\);", body)
    assert body.count("createExecutor(context, index)") == 2
    assert "group.lowerBound.isCurrentRow() && group.upperBound.isCurrentRow()" in body
    assert "new GpuNonFrameOverWindowExec(input, context, spec, group.keys.asList(), reset, dataTypes)" in body


def test_refusals_are_made_at_planner_time():
    g = _code("operator/gpu/GpuSupport.java")
    body = g[g.index("public static boolean nonFrameWindowSupported"):]
    body = body[:body.index("public static boolean sortAggSupported")]
    assert "public static boolean nonFrameWindowSupported(SortWindow window, ExecutionContext context)" in body
    assert "CalciteUtils.getTypes(window.getInput().getRowType())" in body
    # the stock factory's dataTypes.subList(groups.length, ...) slice: aggregate calls whose slot type differs are refused
    assert "dataTypes.get(npart + i)" in body and "dataTypes.get(inputTypes.size() + i)" in body
    assert "window.groups.size() != 1" in body
    assert "first != SqlKind.ROW_NUMBER && first != SqlKind.RANK && first != SqlKind.DENSE_RANK" in body
    assert "GpuAggSpec.tryConvertWindow(calls, inputTypes)" in body
    assert "spec.producesDecimal(inputTypes)" in body and "GpuTypes.supported(inputTypes)" in body
    a = _code("operator/gpu/GpuAggSpec.java")
    w = a[a.index("public static GpuAggSpec tryConvertWindow"):a.index("public boolean producesDecimal")]
    assert "call.filterArg >= 0 || call.isDistinct()" in w
    assert re.search(r"if \(a\.length > 4\)\s*\{\s*return null;", w)
    assert "one.kinds[0] == FIRST_VALUE" in w


def test_natives_are_declared_and_implemented():
    n = _code("operator/gpu/GpuNative.java")
    jni = open(os.path.join(ROOT, "jni", "gsql_jni.c")).read()
    for name in ("windowCreate", "windowApply", "windowDestroy"):
        assert re.search(r"public static native \w+ " + name + r"\(", n), name
        assert re.search(r"NATIVE\(\w+, " + name + r"\)", jni), name
    assert "gsql_window_create(" in jni and "gsql_window_apply(" in jni and "gsql_window_destroy(" in jni


def test_integration_gives_the_planner_patch():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("### Window functions"):]
    sec = sec[:sec.index("\n## ")] if "\n## " in sec else sec
    code = "\n".join(re.findall(r"```java\n(.*?)```", sec, flags=re.S))
    assert "new GpuNonFrameOverWindowExecFactory(" in code
