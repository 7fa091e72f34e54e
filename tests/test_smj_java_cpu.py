"""CPU checks of the Java side of the sort-merge join (the image has no JDK; tests/test_jni_boundary.py already checks every
GpuNative.smj* call site against the declared natives and the shim):

* GpuSortMergeJoinExec extends AbstractExecutor like SortMergeJoinExec, drains the inner input first and keeps the blocked
  and finished rules;
* GpuSortMergeJoinFactory mirrors SortMergeJoinFactory and falls back to the stock SortMergeJoinExec when
  GpuSupport.sortMergeJoinSupported is false;
* sortMergeJoinSupported refuses any other condition and single RIGHT joins, and shares joinSupported's checks;
* the natives are declared and implemented, and INTEGRATION.md gives the visitSortMergeJoin patch."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")


def _code(rel):
    s = re.sub(r"/\*.*?\*/", "", open(os.path.join(PKG, rel)).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def test_executor_extends_what_it_replaces():
    e = _code("operator/GpuSortMergeJoinExec.java")
    assert re.search(r"class GpuSortMergeJoinExec extends AbstractExecutor\s*\{", e)
    assert re.search(r"public GpuSortMergeJoinExec\(Executor outerInput, Executor innerInput, JoinRelType joinType, boolean maxOneRow,\s*"
                     r"List<EquiJoinKey> joinKeys, List<Boolean> keyColumnIsAscending, int\[\] antiOperands,", e)
    body = e[e.index("Chunk doNextChunk()"):]
    assert body.index("innerInput.nextChunk()") < body.index("GpuNative.smjInnerFinish(smj)") < body.index("outerInput.nextChunk()")
    assert "blocked = innerInput.produceIsBlocked();" in e and "blocked = outerInput.produceIsBlocked();" in e
    assert "return outerFinished && left == 0;" in e
    # the releasing smjNext(smj, out, 0) refills `out` with 0 rows: the chunk must be read out of `out` before it
    last = body.index("GpuNative.smjNext(smj, out, (int) Math.min(chunkLimit, left));")
    assert body.index("GpuChunks.toChunk(out, dataTypes, 0, rows)", last) < body.index("GpuNative.smjNext(smj, out, 0)", last)
    assert "ImmutableList.of(innerInput, outerInput)" in e


def test_factory_falls_back_to_the_stock_operator():
    f = _code("mpp/operator/factory/GpuSortMergeJoinFactory.java")
    assert re.search(r"class GpuSortMergeJoinFactory extends ExecutorFactory\b", f)
    assert re.search(r"public GpuSortMergeJoinFactory\(Join join, List<Integer> leftColumns, List<Integer> rightColumns,\s*"
                     r"List<Boolean> columnIsAscending, RexNode otherCond,\s*List<RexNode> operands, boolean maxOneRow, "
                     r"ExecutorFactory inner, ExecutorFactory outer\)", f)
    assert "if (GpuSupport.sortMergeJoinSupported(join, joinKeys, otherCond, maxOneRow, anti ? operands : null, context))" in f
    assert "new GpuSortMergeJoinExec(outer, inner, joinType, maxOneRow, joinKeys, columnIsAscending, antiOperands," in f
    assert re.search(r"new SortMergeJoinExec\(outer, inner, joinType, maxOneRow, joinKeys, columnIsAscending, otherCondition,\s*"
                     r"antiJoinOperands, context\)", f)
    assert "getInputs().get(0).createExecutor(context, index)" in f and "getInputs().get(1).createExecutor(context, index)" in f


def test_support_refuses_conditions_and_shares_join_checks():
    g = _code("operator/gpu/GpuSupport.java")
    body = g[g.index("public static boolean sortMergeJoinSupported"):]
    body = body[:body.index("public static boolean runtimeFilterSupported")]
    assert re.search(r"if \(otherCond != null \|\| \(maxOneRow && join\.getJoinType\(\) == JoinRelType\.RIGHT\)\)\s*\{\s*return false;", body)
    assert "return joinSupported(join, keys, null, maxOneRow, antiOperands, context);" in body


def test_jni_checks_the_key_array_lengths():
    jni = open(os.path.join(ROOT, "jni", "gsql_jni.c")).read()
    body = jni[jni.index("NATIVE(jlong, smjCreate)"):]
    body = body[:body.index("\n}\n")]
    assert "desc[GSQL_MAX_KEYS] = {0}" in body
    for a in ("innerKeys", "keyTypes", "keyDesc"):
        assert f"(*env)->GetArrayLength(env, {a}) != nk" in body
    assert body.index("throw_status(env, NULL, GSQL_E_INVALID)") < body.index("gsql_smj_create(")


def test_natives_are_declared_and_implemented():
    n = _code("operator/gpu/GpuNative.java")
    jni = open(os.path.join(ROOT, "jni", "gsql_jni.c")).read()
    for name in ("smjCreate", "smjInnerConsume", "smjInnerFinish", "smjProbe", "smjNext", "smjDestroy"):
        assert re.search(r"public static native \w+ " + name + r"\(", n), name
        assert re.search(r"NATIVE\(\w+, " + name + r"\)", jni), name


def test_integration_gives_the_planner_patch():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = doc[doc.index("### Sort-merge join"):]
    sec = sec[:sec.index("\n## ")] if "\n## " in sec else sec
    code = "\n".join(re.findall(r"```java\n(.*?)```", sec, flags=re.S))
    assert "visitSortMergeJoin" in code and "new GpuSortMergeJoinFactory(" in code
    assert "separate exchanges or sources" in sec
