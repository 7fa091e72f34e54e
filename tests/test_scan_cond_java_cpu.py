"""CPU checks, by text (the image has no JDK), of GpuExpression's CASE / COALESCE / IN / BETWEEN / DATE translation: what
it accepts and refuses is what tests/scan_cond_ref.py restates; tests/test_jni_boundary.py checks the scanCreate2 native
against the shim and its call site."""
import os
import re

from tests import scan_cond_ref as Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GPU = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor", "operator", "gpu")


def _code(name):
    s = re.sub(r"/\*.*?\*/", "", open(os.path.join(GPU, name)).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def _method(src, start):
    body = src[src.index(start):]
    depth, i = 0, body.index("{")
    for k in range(i, len(body)):
        depth += {"{": 1, "}": -1}.get(body[k], 0)
        if depth == 0:
            return body[:k + 1]
    raise AssertionError(start)


def test_in_and_between_only_over_a_bare_integer_column_and_at_most_100_constants():
    g = _code("GpuExpression.java")
    assert "MAX_IN_CONSTANTS = 100" in g and Q.REF_MAX_IN_CONSTANTS == 100
    body = _method(g, "private static GpuExpression setTest(")
    # IN over an expression: refused (the reference reads the computed value under a NULL flag)
    assert "!(x instanceof RexInputRef) || constants.isEmpty() || constants.size() > MAX_IN_CONSTANTS" in body
    assert "GpuTypes.code(inputTypes.get(i)) == GpuNative.T_FP64" in body and "!GpuTypes.isNumeric(inputTypes.get(i))" in body
    assert "if (!(constants.get(k) instanceof RexLiteral))" in body
    assert "anyNull ? nullOf(GpuNative.T_INT64) : col(i).withPool(op, values)" in body    # a NULL constant: every row NULL
    t = _code("GpuExpression.java")
    t = t[t.index("private static GpuExpression translate("):]
    assert "case IN:" in t and "SqlKind.ROW" in t and "setTest(operands.get(0), list, OP_IN, inputTypes)" in t
    assert "setTest(operands.get(0), operands.subList(1, 3), OP_BETWEEN, inputTypes)" in t


def test_date_comparison_packs_a_char_constant_and_refuses_other_forms():
    g = _code("GpuExpression.java")
    body = _method(g, "private static GpuExpression dateComparison(")
    for kind in ("LESS_THAN", "LESS_THAN_OR_EQUAL", "GREATER_THAN", "GREATER_THAN_OR_EQUAL", "EQUALS", "NOT_EQUALS"):
        assert "case %s:" % kind in body
    # column on the left, a literal on the right, a DATE column (not DATETIME), a CHAR literal (not a DATE-typed one)
    assert "!(operands.get(0) instanceof RexInputRef) || !(operands.get(1) instanceof RexLiteral)" in body
    assert "getDataClass() != java.sql.Date.class" in body
    assert "lit.getType().getSqlTypeName() != SqlTypeName.CHAR" in body
    # the constant: TimeStorage.writeDate(DateType.convertFrom(literal)); a NULL literal: every row NULL
    assert "DataTypes.DateType.convertFrom(lit.getValueAs(String.class))" in body
    assert "lit(TimeStorage.writeDate(((OriginalDate) date).getMysqlDateTime()))" in body
    assert "col(i).binary(op, nullOf(GpuNative.T_INT64))" in body
    assert Q.write_date(1995, 3, 15) == 1825257471829082112
    # a DATE column anywhere else inside an expression stays refused
    assert "GpuTypes.isNumeric(inputTypes.get(i)) ? col(i) : null; " in open(os.path.join(GPU, "GpuExpression.java")).read()


def test_case_and_coalesce_branches_must_have_the_call_type():
    g = _code("GpuExpression.java")
    br = _method(g, "private static GpuExpression branch(")
    assert "t != SqlTypeName.BIGINT && t != SqlTypeName.DOUBLE" in br
    assert "node.getType().getSqlTypeName() != t" in br and "x.resultType(inputTypes) == code" in br
    assert "return nullOf(code);" in br                                                  # a missing ELSE / NULL branch
    case = _method(g, "private static GpuExpression caseOf(")
    assert "operands.size() % 2 == 0" in case                                            # Calcite always gives the ELSE
    assert "acc.then(cond, 0).then(value, OP_CASE_WHEN)" in case                         # right to left
    assert "for (int i = operands.size() - 3; i >= 0 && acc != null; i -= 2)" in case
    t = g[g.index("private static GpuExpression translate("):]
    assert "acc == null ? x : acc.binary(OP_COALESCE, x)" in t


def test_programs_are_refused_past_the_operand_stack():
    g = _code("GpuExpression.java")
    assert "e != null && e.fits() && e.resultType(inputTypes) >= 0 ? e : null" in g
    rt = _method(g, "int resultType(List<DataType> inputTypes)")
    assert "if (sp == MAX_STACK)" in rt and "MAX_STACK = 4" in g


def test_executor_picks_create2_for_the_new_ops():
    e = re.sub(r"//[^\n]*", "", open(os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor", "operator",
                                                  "GpuVectorizedFilterProjectExec.java")).read())
    assert "create2 |= outputs[i].needsCreate2();" in e and "GpuNative.scanCreate2(ctx, inputCodes," in e
    g = _code("GpuExpression.java")
    assert "if (op >= OP_CONST_NULL)" in _method(g, "public boolean needsCreate2()")
    shim = open(os.path.join(ROOT, "jni", "gsql_jni.c")).read()
    assert "gsql_scan_create2((gsql_ctx *)(intptr_t)ctx, s, pool, npool, &sc)" in shim
    assert "e->ins[i].arg += *npool;" in shim
