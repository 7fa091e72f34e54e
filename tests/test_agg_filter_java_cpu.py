"""CPU checks of the Java planner's decisions for the hash aggregation's FILTER argument and input types (the image has no
JDK; the checks read the sources):

* GpuAggSpec.tryConvert returns null for a call whose FILTER column is not INT / BIGINT / DOUBLE: a DATE / DATETIME /
  TIMESTAMP column would reach the kernels as its packed BIGINT and filter rows on values below 1, while the stock
  AggOpenHashMap.putChunk filters on Long cells only (a Date / Timestamp never filters);
* GpuSupport.aggShapeSupported requires a GPU type for every input column, which is what GpuTypes.codes(inputTypes) in
  GpuHashAggExec and GpuSortAggExec assumes (it throws otherwise), so such plans keep the stock operator;
* INTEGRATION.md states both rules."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")


def _code(rel):
    s = re.sub(r"/\*.*?\*/", "", open(os.path.join(PKG, rel)).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def _method(src, signature):
    """The body of the method whose declaration starts with `signature` (brace-matched)."""
    i = src.index(signature)
    j = src.index("{", i)
    depth = 0
    for k in range(j, len(src)):
        depth += {"{": 1, "}": -1}.get(src[k], 0)
        if depth == 0:
            return src[j:k + 1]
    raise AssertionError(f"unbalanced braces after {signature}")


def test_try_convert_refuses_a_non_numeric_filter_column():
    body = _method(_code("operator/gpu/GpuAggSpec.java"), "public static GpuAggSpec tryConvert(")
    check = re.search(r"if \(call\.filterArg >= 0 && !GpuTypes\.isNumeric\(inputTypes\.get\(call\.filterArg\)\)\)\s*\{\s*"
                      r"return null;\s*\}", body)
    assert check, body
    assert check.start() < body.index("filters[i] = call.filterArg;")      # decided before the filter is passed on
    assert body.index("for (int i = 0; i < n; i++)") < check.start()       # for every call


def test_is_numeric_excludes_packed_time_and_types_without_a_gpu_form():
    t = _code("operator/gpu/GpuTypes.java")
    assert re.search(r"public static boolean isNumeric\(DataType type\)\s*\{\s*return code\(type\) >= 0 && !isPackedTime\(type\);", t)
    packed = _method(t, "public static boolean isPackedTime(")
    assert "java.sql.Date.class" in packed and "java.sql.Timestamp.class" in packed
    code = _method(t, "public static int code(")
    assert "if (isPackedTime(type))" in code and "return GpuNative.T_INT64;" in code   # why isNumeric, not code() >= 0


def test_agg_shape_requires_every_input_column_to_have_a_gpu_type():
    g = _code("operator/gpu/GpuSupport.java")
    shape = _method(g, "private static boolean aggShapeSupported(")
    assert re.search(r"if \(!GpuTypes\.supported\(inputTypes\)\)\s*\{\s*return false;\s*\}", shape), shape
    assert shape.index("GpuTypes.supported(inputTypes)") < shape.index("GpuAggSpec.tryConvert(calls, inputTypes)")
    # both hash and sorted aggregation go through it, with the executors' input types
    for m in ("public static boolean aggSupported(", "public static boolean sortAggSupported("):
        assert "return aggShapeSupported(agg.getGroupSet(), agg.getRowType(), agg.getAggCallList(), inputTypes, context);" \
            in _method(g, m), m
    assert "GpuSupport.sortAggSupported(sortAgg, input.getDataTypes(), context)" in _code("mpp/operator/factory/GpuSortAggExecFactory.java")


def test_executors_stage_every_input_column():
    """The assumption aggShapeSupported now checks: both executors map the whole input row to GPU type codes."""
    assert "this.inputCodes = GpuTypes.codes(inputTypes);" in _code("operator/GpuHashAggExec.java")
    assert "this.inputCodes = GpuTypes.codes(input.getDataTypes());" in _code("operator/GpuSortAggExec.java")
    t = _method(_code("operator/gpu/GpuTypes.java"), "public static int[] codes(")
    assert "throw new GpuExecutorException(" in t


def test_integration_states_the_filter_and_input_type_rules():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("`GpuSupport` mirrors the `GSQL_E_UNSUPPORTED` rules"):]
    sec = sec[:sec.index("\n\n")]
    assert "every input column" in sec
    assert "FILTER" in sec and "DATE" in sec and "`GpuAggSpec.tryConvert`" in sec
