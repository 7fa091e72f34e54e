"""CPU checks of the Java side of the grouping-sets aggregation (the image has no JDK; tests/test_jni_boundary.py checks
every GpuNative.gsAgg* call site against the declared natives and the shim, and compiles and links the shim):

* GpuExpandHashAggExec is a consumer like GpuHashAggExec and drives gsql_gsagg through the gsAgg* natives;
* GpuExpandHashAggExecutorFactory takes HashAggExecutorFactory's arguments plus the LogicalExpand;
* GpuSupport.groupingSetsSupported restates gsql_gsagg_create's refusals and expandItems the accepted item forms;
* INTEGRATION.md's visitHashAgg patch applies only to a partial agg or a pipeline of parallelism 1."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")


def _code(rel):
    s = re.sub(r"/\*.*?\*/", "", open(os.path.join(PKG, rel)).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def _method(src, start):
    body = src[src.index(start):]
    depth, i = 0, body.index("{")
    for k in range(i, len(body)):
        depth += {"{": 1, "}": -1}.get(body[k], 0)
        if depth == 0:
            return body[:k + 1]
    raise AssertionError(start)


def test_executor_drives_the_gsagg_natives():
    e = _code("operator/GpuExpandHashAggExec.java")
    assert re.search(r"class GpuExpandHashAggExec extends AbstractExecutor implements ConsumerExecutor\s*\{", e)
    assert "GpuNative.gsAggCreate(ctx, inputCodes, expandCodes, projSrc, projCol, projValue, groups, spec.kinds, spec.cols," in e
    for call in ("GpuNative.gsAggConsume(agg, in);", "GpuNative.gsAggFinish(agg);", "GpuNative.gsAggNext(agg, out, chunkLimit);",
                 "GpuNative.gsAggDestroy(agg);", "GpuChunks.append(in, chunk, inputCodes);"):
        assert call in e, call
    assert "this.inputCodes = GpuTypes.codes(inputTypes);" in e and "this.expandCodes = GpuTypes.codes(expandColumns);" in e


def test_factory_builds_from_the_expand():
    f = _code("mpp/operator/factory/GpuExpandHashAggExecutorFactory.java")
    assert re.search(r"class GpuExpandHashAggExecutorFactory extends ExecutorFactory\b", f)
    assert ("public GpuExpandHashAggExecutorFactory(HashAgg hashAgg, LogicalExpand expand, int parallelism, int taskNumber,\n"
            "                                           Integer rowCount, List<DataType> inputDataTypes)") in f
    assert "GpuAggSpec.tryConvert(hashAgg.getAggCallList(), expandDataTypes)" in f
    assert "GpuSupport.expandItems(expand)" in f and "CalciteUtils.getTypes(expand.getRowType())" in f


def test_support_restates_the_refusals():
    g = _code("operator/gpu/GpuSupport.java")
    items = _method(g, "public static ExpandItems expandItems(LogicalExpand expand)")
    assert "n instanceof RexInputRef" in items and "RexLiteral.isNullLiteral(n)" in items
    assert "SqlTypeName.INT_TYPES.contains(n.getType().getSqlTypeName())" in items
    assert re.search(r"\} else \{\s*return null;", items)                       # any other expression: stock operators
    body = _method(g, "public static boolean groupingSetsSupported(HashAgg agg, LogicalExpand expand, List<DataType> inputTypes,")
    assert "it.src.length < 1 || it.src.length > MAX_SETS" in body and "static final int MAX_SETS = 16;" in g
    assert "aggShapeSupported(agg.getGroupSet(), agg.getRowType(), agg.getAggCallList(), outTypes, context)" in body
    assert "call.getAggregation().getKind() == SqlKind.__FIRST_VALUE" in body
    assert "it.src[s][c] != GpuNative.EXPAND_INPUT || it.col[s][c] != it.col[0][c]" in body        # same input in every set
    assert "call.filterArg >= 0" in body                                                           # FILTER columns too
    assert "GpuTypes.code(in) != code || in.getDataClass() != outTypes.get(c).getDataClass()" in body
    assert "code == GpuNative.T_FP64" in body and "Integer.MIN_VALUE" in body                      # constants
    assert "distinct = it.value[q][g] != it.value[s][g];" in body                                  # the $e column
    n = _code("operator/gpu/GpuNative.java")
    assert "EXPAND_INPUT = 0, EXPAND_NULL = 1, EXPAND_CONST = 2" in n


def test_integration_patch_is_partial_or_single_pipeline_only():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("### Grouping sets"):]
    sec = sec[:sec.index("\n### ")]
    code = "\n".join(re.findall(r"```java\n(.*?)```", sec, flags=re.S))
    assert "visitHashAgg" in code
    assert "agg.getInput() instanceof LogicalExpand && (agg.isPartial() || pipelineFragment.getParallelism() == 1)" in code
    assert "GpuSupport.groupingSetsSupported(agg, expand, inputColumns, context)" in code
    assert "visit(expand, expand.getInput(), childFragment)" in code
    assert "new GpuExpandHashAggExecutorFactory(agg, expand," in code
    assert "LocalExchangeMode.PARTITION" not in code      # expanded rows' (keys, $e) partitioning cannot route input rows
