"""CPU checks of the Java side of the sorted aggregation (the image has no JDK; tests/test_jni_boundary.py already checks
every GpuNative.sortAgg* call site against the declared natives and the shim):

* GpuSortAggExec extends AbstractExecutor like SortAggExec and keeps its constructor's arguments;
* GpuSortAggExecFactory mirrors SortAggExecFactory and falls back to the stock SortAggExec when
  GpuSupport.sortAggSupported is false;
* sortAggSupported refuses FILTER arguments and shares aggSupported's checks;
* the natives are declared and implemented, and INTEGRATION.md gives the planner patch for both branches of visitSortAgg."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")


def _code(rel):
    s = re.sub(r"/\*.*?\*/", "", open(os.path.join(PKG, rel)).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def test_executor_extends_what_it_replaces():
    e = _code("operator/GpuSortAggExec.java")
    assert re.search(r"class GpuSortAggExec extends AbstractExecutor\s*\{", e)
    assert re.search(r"public GpuSortAggExec\(Executor input, int\[\] groups, GpuAggSpec spec, List<DataType> outputColumnMeta,\s*"
                     r"ExecutionContext context\)", e)
    assert "GpuChunks.append(in, chunk, inputCodes);" in e
    assert "blocked = input.produceIsBlocked();" in e and "inputFinished = input.produceIsFinished();" in e


def test_factory_falls_back_to_the_stock_operator():
    f = _code("mpp/operator/factory/GpuSortAggExecFactory.java")
    assert re.search(r"class GpuSortAggExecFactory extends ExecutorFactory\b", f)
    assert "public GpuSortAggExecFactory(SortAgg sortAgg, ExecutorFactory executorFactory, int parallelism)" in f
    assert "if (GpuSupport.sortAggSupported(sortAgg, input.getDataTypes(), context))" in f
    assert "new GpuSortAggExec(input, groups, spec, outputDataTypes, context)" in f
    assert "new SortAggExec(input, groups, aggregators, outputDataTypes, context)" in f
    assert "AggregateUtils.convertAggregators(input.getDataTypes()" in f
    assert "getInputs().get(0).createExecutor(context, k)" in f


def test_filter_arguments_are_refused_and_agg_checks_shared():
    g = _code("operator/gpu/GpuSupport.java")
    body = g[g.index("public static boolean sortAggSupported"):]
    body = body[:body.index("private static boolean aggShapeSupported")]
    assert re.search(r"if \(call\.filterArg >= 0\)\s*\{\s*return false;", body)
    assert "return aggShapeSupported(agg.getGroupSet(), agg.getRowType(), agg.getAggCallList(), inputTypes, context);" in body
    agg = g[g.index("public static boolean aggSupported"):g.index("public static boolean sortAggSupported")]
    assert "return aggShapeSupported(agg.getGroupSet(), agg.getRowType(), agg.getAggCallList(), inputTypes, context);" in agg
    shape = g[g.index("private static boolean aggShapeSupported"):]
    assert "GpuAggSpec.tryConvert(calls, inputTypes)" in shape and "!spec.producesDecimal(inputTypes)" in shape


def test_natives_are_declared_and_implemented():
    n = _code("operator/gpu/GpuNative.java")
    jni = open(os.path.join(ROOT, "jni", "gsql_jni.c")).read()
    for name in ("sortAggCreate", "sortAggConsume", "sortAggFinish", "sortAggNext", "sortAggDestroy"):
        assert re.search(r"public static native \w+ " + name + r"\(", n), name
        assert "NATIVE(" in jni and re.search(r"NATIVE\(\w+, " + name + r"\)", jni), name


def test_integration_gives_the_planner_patch_for_both_branches():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("### Sorted aggregation"):]
    sec = sec[:sec.index("\n## ")] if "\n## " in sec else sec
    code = "\n".join(re.findall(r"```java\n(.*?)```", sec, flags=re.S))
    assert "visitSortAgg" in code
    assert code.count("new GpuSortAggExecFactory(") >= 2
