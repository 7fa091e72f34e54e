/*
 * A scalar expression as the postfix program gsql_scan_* evaluates (include/gsql_gpu.h: gsql_expr, gsql_expr_op): the
 * GPU-side stand-in for a VectorizedExpression tree (executor/vectorized/**).  Programs are immutable; the builder
 * methods return new programs.  fromRex() translates the RexNode the planner hands to VectorizedExpressionBuilder and
 * returns null for anything the GPU path does not evaluate (the factory then keeps the stock operator).
 */
package com.alibaba.polardbx.executor.operator.gpu;

import com.alibaba.polardbx.common.utils.time.core.OriginalDate;
import com.alibaba.polardbx.common.utils.time.core.TimeStorage;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.alibaba.polardbx.optimizer.core.datatype.DataTypes;
import org.apache.calcite.rex.RexCall;
import org.apache.calcite.rex.RexInputRef;
import org.apache.calcite.rex.RexLiteral;
import org.apache.calcite.rex.RexNode;
import org.apache.calcite.sql.SqlKind;
import org.apache.calcite.sql.type.SqlTypeName;

import java.math.BigDecimal;
import java.util.ArrayList;
import java.util.Arrays;
import java.util.List;

public final class GpuExpression {
    // gsql_expr_op
    public static final int OP_COL = 1, OP_CONST_I64 = 2, OP_CONST_F64 = 3, OP_ADD = 4, OP_SUB = 5, OP_MUL = 6, OP_DIV = 7, OP_NEG = 8,
        OP_LT = 9, OP_LE = 10, OP_GT = 11, OP_GE = 12, OP_EQ = 13, OP_NE = 14, OP_AND = 15, OP_OR = 16, OP_NOT = 17, OP_IS_NULL = 18,
        OP_CAST_F64 = 19, OP_CAST_I64 = 20,
        OP_CONST_NULL = 32, OP_CASE_WHEN = 33, OP_COALESCE = 34, OP_BETWEEN = 35, OP_IN = 36;
    /** GSQL_MAX_EXPR_INS */
    public static final int MAX_INSTRUCTIONS = 24;
    /** GSQL_MAX_EXPR_STACK */
    public static final int MAX_STACK = 4;
    /** The reference generates IN classes for 1..100 constants (codegen/data/InColConstOperators.tdd). */
    public static final int MAX_IN_CONSTANTS = 100;

    public final int[] ops;
    public final int[] args;
    /** constants: the long value, or Double.doubleToRawLongBits for OP_CONST_F64 */
    public final long[] consts;
    /** IN lists and BETWEEN bounds: OP_IN / OP_BETWEEN's arg is an offset into this program's pool */
    public final long[] pool;

    private GpuExpression(int[] ops, int[] args, long[] consts, long[] pool) {
        this.ops = ops;
        this.args = args;
        this.consts = consts;
        this.pool = pool;
    }

    private static GpuExpression one(int op, int arg, long k) {
        return new GpuExpression(new int[] {op}, new int[] {arg}, new long[] {k}, new long[0]);
    }

    /** NULL of a BIGINT (GpuNative.T_INT64) or DOUBLE (GpuNative.T_FP64) */
    public static GpuExpression nullOf(int type) {
        return one(OP_CONST_NULL, type, 0);
    }

    /** true if the program holds an op only gsql_scan_create2 accepts (GpuNative.scanCreate2) */
    public boolean needsCreate2() {
        for (int op : ops) {
            if (op >= OP_CONST_NULL) {
                return true;
            }
        }
        return false;
    }

    public static GpuExpression col(int index) {
        return one(OP_COL, index, 0);
    }

    public static GpuExpression lit(long v) {
        return one(OP_CONST_I64, 0, v);
    }

    public static GpuExpression lit(double v) {
        return one(OP_CONST_F64, 0, Double.doubleToRawLongBits(v));
    }

    /** this program, then other's (if any), then op (if not 0) */
    private GpuExpression then(GpuExpression other, int op) {
        int n = ops.length + (other == null ? 0 : other.ops.length) + (op == 0 ? 0 : 1);
        int[] o = new int[n];
        int[] a = new int[n];
        long[] k = new long[n];
        System.arraycopy(ops, 0, o, 0, ops.length);
        System.arraycopy(args, 0, a, 0, ops.length);
        System.arraycopy(consts, 0, k, 0, ops.length);
        long[] p = pool;
        if (other != null) {
            System.arraycopy(other.ops, 0, o, ops.length, other.ops.length);
            System.arraycopy(other.args, 0, a, ops.length, other.ops.length);
            System.arraycopy(other.consts, 0, k, ops.length, other.ops.length);
            for (int i = ops.length; i < ops.length + other.ops.length; i++) {
                if (o[i] == OP_IN || o[i] == OP_BETWEEN) {
                    a[i] += pool.length; // the right operand's pool follows this one's
                }
            }
            p = Arrays.copyOf(pool, pool.length + other.pool.length);
            System.arraycopy(other.pool, 0, p, pool.length, other.pool.length);
        }
        if (op != 0) {
            o[n - 1] = op;
        }
        return new GpuExpression(o, a, k, p);
    }

    /** x IN (values) / x BETWEEN lo AND hi: the constants go to the pool */
    private GpuExpression withPool(int op, long[] values) {
        GpuExpression e = then(null, op);
        e.args[e.ops.length - 1] = pool.length;
        e.consts[e.ops.length - 1] = op == OP_IN ? values.length : 0;
        long[] p = Arrays.copyOf(pool, pool.length + values.length);
        System.arraycopy(values, 0, p, pool.length, values.length);
        return new GpuExpression(e.ops, e.args, e.consts, p);
    }

    public GpuExpression binary(int op, GpuExpression right) {
        return then(right, op);
    }

    public GpuExpression unary(int op) {
        return then(null, op);
    }

    public boolean fits() {
        return ops.length <= MAX_INSTRUCTIONS;
    }

    /**
     * The program's stack walk as gsql_scan_create2 type-checks it: GpuNative.T_INT64 or T_FP64 for the result, -1 if the
     * operand stack would grow past MAX_STACK or CASE / COALESCE would join an integer and a double.
     */
    int resultType(List<DataType> inputTypes) {
        boolean[] isf = new boolean[MAX_INSTRUCTIONS + 1];
        int sp = 0;
        for (int i = 0; i < ops.length; i++) {
            int op = ops[i];
            if (op == OP_COL || op == OP_CONST_I64 || op == OP_CONST_F64 || op == OP_CONST_NULL) {
                if (sp == MAX_STACK) {
                    return -1;
                }
                isf[sp++] = op == OP_CONST_F64 || (op == OP_CONST_NULL && args[i] == GpuNative.T_FP64) || (op == OP_COL && GpuTypes.code(inputTypes.get(args[i])) == GpuNative.T_FP64);
            } else if (op == OP_CASE_WHEN) {
                if (sp < 3 || isf[sp - 2] || isf[sp - 3] != isf[sp - 1]) {
                    return -1;
                }
                sp -= 2;
            } else if (op == OP_COALESCE) {
                if (sp < 2 || isf[sp - 2] != isf[sp - 1]) {
                    return -1;
                }
                sp--;
            } else if (op == OP_NEG || op == OP_CAST_F64 || op == OP_CAST_I64 || op == OP_NOT || op == OP_IS_NULL || op == OP_IN
                || op == OP_BETWEEN) {
                if (sp < 1) {
                    return -1;
                }
                isf[sp - 1] = op == OP_CAST_F64 || (op == OP_NEG && isf[sp - 1]);
            } else {
                if (sp < 2) {
                    return -1;
                }
                sp--;
                isf[sp - 1] = op >= OP_ADD && op <= OP_DIV && (isf[sp - 1] || isf[sp] || op == OP_DIV);
            }
        }
        return sp != 1 ? -1 : isf[0] ? GpuNative.T_FP64 : GpuNative.T_INT64;
    }

    /**
     * RexNode -> program.  Covered: input refs over INT / BIGINT / DOUBLE columns, exact and approximate numeric
     * literals, + - * unary minus, `/` where the planner typed the quotient DOUBLE, the six comparisons, AND / OR / NOT,
     * IS NULL / IS NOT NULL, CAST to BIGINT / SIGNED / DOUBLE; CASE and COALESCE whose branches all have the call's BIGINT
     * or DOUBLE type; IN (1..100 integer constants) and BETWEEN over a bare INT / BIGINT column; a DATE column compared
     * with a CHAR constant (the packed long of its date).  Programs deeper than the GPU's operand stack are refused.
     */
    public static GpuExpression fromRex(RexNode node, List<DataType> inputTypes) {
        if (node instanceof RexInputRef) { // a bare column passes through whatever its block type (DATE / DATETIME as packed longs)
            int i = ((RexInputRef) node).getIndex();
            return i < inputTypes.size() && GpuTypes.code(inputTypes.get(i)) >= 0 ? col(i) : null;
        }
        GpuExpression e = translate(node, inputTypes);
        return e != null && e.fits() && e.resultType(inputTypes) >= 0 ? e : null;
    }

    private static GpuExpression translate(RexNode node, List<DataType> inputTypes) {
        if (node instanceof RexInputRef) {
            int i = ((RexInputRef) node).getIndex();
            return i < inputTypes.size() && GpuTypes.isNumeric(inputTypes.get(i)) ? col(i) : null; // inside an expression: numbers only
        }
        if (node instanceof RexLiteral) {
            Object v = ((RexLiteral) node).getValue3();
            if (v instanceof BigDecimal) {
                BigDecimal d = (BigDecimal) v;
                return d.scale() <= 0 && d.abs().compareTo(BigDecimal.valueOf(Long.MAX_VALUE)) <= 0 ? lit(d.longValueExact()) : lit(d.doubleValue());
            }
            if (v instanceof Long || v instanceof Integer) {
                return lit(((Number) v).longValue());
            }
            if (v instanceof Double || v instanceof Float) {
                return lit(((Number) v).doubleValue());
            }
            return null;
        }
        if (!(node instanceof RexCall)) {
            return null;
        }
        RexCall call = (RexCall) node;
        List<RexNode> operands = call.getOperands();
        GpuExpression date = dateComparison(call, inputTypes);
        if (date != null) {
            return date;
        }
        int op;
        switch (call.getKind()) {
        case PLUS: op = OP_ADD; break;
        case MINUS: op = OP_SUB; break;
        case TIMES: op = OP_MUL; break;
        case DIVIDE: {
            // OP_DIV is the DOUBLE division (NULL on a zero divisor).  The reference types `/` DOUBLE only when an operand is
            // approximate; integer / integer is DECIMAL there and stays on the stock operator.
            String result = call.getType().getSqlTypeName().getName();
            if (!"DOUBLE".equals(result) && !"FLOAT".equals(result)) {
                return null;
            }
            op = OP_DIV;
            break;
        }
        case LESS_THAN: op = OP_LT; break;
        case LESS_THAN_OR_EQUAL: op = OP_LE; break;
        case GREATER_THAN: op = OP_GT; break;
        case GREATER_THAN_OR_EQUAL: op = OP_GE; break;
        case EQUALS: op = OP_EQ; break;
        case NOT_EQUALS: op = OP_NE; break;
        case AND: op = OP_AND; break;
        case OR: op = OP_OR; break;
        case NOT: return unaryOf(operands, inputTypes, OP_NOT);
        case MINUS_PREFIX: return unaryOf(operands, inputTypes, OP_NEG);
        case IS_NULL: return unaryOf(operands, inputTypes, OP_IS_NULL);
        case IS_NOT_NULL: {
            GpuExpression x = unaryOf(operands, inputTypes, OP_IS_NULL);
            return x == null ? null : x.unary(OP_NOT);
        }
        case CAST: {
            // the targets Rex2VectorizedExpressionVisitor.VECTORIZED_CAST_FUNCTION_NAMES vectorises: CastToDouble, and
            // CastToSigned ((long) Math.rint(x) of a double); INTEGER and FLOAT targets are not among them
            String target = call.getType().getSqlTypeName().getName();
            if ("DOUBLE".equals(target)) {
                return unaryOf(operands, inputTypes, OP_CAST_F64);
            }
            if ("BIGINT".equals(target) || "SIGNED".equals(target)) {
                return unaryOf(operands, inputTypes, OP_CAST_I64);
            }
            return null;
        }
        case CASE: return caseOf(call, inputTypes);
        case COALESCE: {
            GpuExpression acc = null;
            for (RexNode o : operands) { // folded left: the first non-NULL argument
                GpuExpression x = branch(o, call, inputTypes);
                if (x == null) {
                    return null;
                }
                acc = acc == null ? x : acc.binary(OP_COALESCE, x);
            }
            return acc;
        }
        case IN: {
            // the reference vectorises IN only as (column, constants...): Rex2VectorizedExpressionVisitor.rewrite flattens
            // ROW(constants) into the call (AbstractIn{Integer,Long}ColLongConstVectorizedExpression)
            List<RexNode> list = new ArrayList<>(operands.subList(1, operands.size()));
            if (list.size() == 1 && list.get(0) instanceof RexCall && list.get(0).getKind() == SqlKind.ROW) {
                list = ((RexCall) list.get(0)).getOperands();
            }
            return setTest(operands.get(0), list, OP_IN, inputTypes);
        }
        case BETWEEN: return operands.size() == 3 ? setTest(operands.get(0), operands.subList(1, 3), OP_BETWEEN, inputTypes) : null;
        default: return null;
        }
        if (operands.size() < 2) {
            return null;
        }
        GpuExpression acc = translate(operands.get(0), inputTypes);
        for (int i = 1; i < operands.size() && acc != null; i++) { // n-ary AND / OR / + / * fold left to right
            GpuExpression right = translate(operands.get(i), inputTypes);
            acc = right == null ? null : acc.binary(op, right);
        }
        return acc;
    }

    /**
     * CASE WHEN c1 THEN v1 ... ELSE e END (CaseVectorizedExpression: the first TRUE condition wins), compiled right to left
     * as e, cn, vn, CASE_WHEN, ..., c1, v1, CASE_WHEN.  Calcite gives a CASE without ELSE a NULL literal.
     */
    private static GpuExpression caseOf(RexCall call, List<DataType> inputTypes) {
        List<RexNode> operands = call.getOperands();
        if (operands.size() < 3 || operands.size() % 2 == 0) {
            return null;
        }
        GpuExpression acc = branch(operands.get(operands.size() - 1), call, inputTypes);
        for (int i = operands.size() - 3; i >= 0 && acc != null; i -= 2) {
            GpuExpression cond = translate(operands.get(i), inputTypes);
            GpuExpression value = branch(operands.get(i + 1), call, inputTypes);
            acc = cond == null || value == null ? null : acc.then(cond, 0).then(value, OP_CASE_WHEN);
        }
        return acc;
    }

    /**
     * A CASE / COALESCE branch: only one that already has the call's type (BIGINT or DOUBLE), since the reference's
     * branch vectors are copied into the result vector unconverted; a NULL literal is the NULL of that type.
     */
    private static GpuExpression branch(RexNode node, RexCall call, List<DataType> inputTypes) {
        SqlTypeName t = call.getType().getSqlTypeName();
        if (t != SqlTypeName.BIGINT && t != SqlTypeName.DOUBLE) {
            return null;
        }
        int code = t == SqlTypeName.DOUBLE ? GpuNative.T_FP64 : GpuNative.T_INT64;
        if (node instanceof RexLiteral && ((RexLiteral) node).getValue3() == null) {
            return nullOf(code);
        }
        if (node.getType().getSqlTypeName() != t) {
            return null;
        }
        GpuExpression x = translate(node, inputTypes);
        return x != null && x.resultType(inputTypes) == code ? x : null;
    }

    /**
     * IN / BETWEEN over a bare INT / BIGINT column: the reference compares the value a NULL row's block holds (0) without
     * merging the NULL flag, as GSQL_OP_IN / GSQL_OP_BETWEEN do; over an expression it would read the computed value under
     * the flag, which the GPU does not keep, so that form is refused.  Any NULL constant makes every row NULL.
     */
    private static GpuExpression setTest(RexNode x, List<RexNode> constants, int op, List<DataType> inputTypes) {
        if (!(x instanceof RexInputRef) || constants.isEmpty() || constants.size() > MAX_IN_CONSTANTS) {
            return null;
        }
        int i = ((RexInputRef) x).getIndex();
        if (i >= inputTypes.size() || !GpuTypes.isNumeric(inputTypes.get(i)) || GpuTypes.code(inputTypes.get(i)) == GpuNative.T_FP64) {
            return null;
        }
        long[] values = new long[constants.size()];
        boolean anyNull = false;
        for (int k = 0; k < values.length; k++) {
            if (!(constants.get(k) instanceof RexLiteral)) {
                return null;
            }
            Object v = ((RexLiteral) constants.get(k)).getValue3();
            if (v == null) {
                anyNull = true;
            } else if (v instanceof BigDecimal && ((BigDecimal) v).scale() <= 0
                && ((BigDecimal) v).abs().compareTo(BigDecimal.valueOf(Long.MAX_VALUE)) <= 0) {
                values[k] = ((BigDecimal) v).longValueExact();
            } else if (v instanceof Long || v instanceof Integer) {
                values[k] = ((Number) v).longValue();
            } else {
                return null;
            }
        }
        return anyNull ? nullOf(GpuNative.T_INT64) : col(i).withPool(op, values);
    }

    /**
     * DATE column <cmp> CHAR constant: ComparisonBinaryDateColumnConst compares the DateBlock's packed longs with
     * TimeStorage.writeDate(DateType.convertFrom(constant)), NULL merged from the column; a NULL constant makes every row
     * NULL.  Only this form: a DATE-typed literal binds no vectorised class, the constant must be on the right, and
     * DATE col vs DATE col reads its right operand at the wrong position under a selection.  null: not this form.
     */
    private static GpuExpression dateComparison(RexCall call, List<DataType> inputTypes) {
        int op;
        switch (call.getKind()) {
        case LESS_THAN: op = OP_LT; break;
        case LESS_THAN_OR_EQUAL: op = OP_LE; break;
        case GREATER_THAN: op = OP_GT; break;
        case GREATER_THAN_OR_EQUAL: op = OP_GE; break;
        case EQUALS: op = OP_EQ; break;
        case NOT_EQUALS: op = OP_NE; break;
        default: return null;
        }
        List<RexNode> operands = call.getOperands();
        if (operands.size() != 2 || !(operands.get(0) instanceof RexInputRef) || !(operands.get(1) instanceof RexLiteral)) {
            return null;
        }
        int i = ((RexInputRef) operands.get(0)).getIndex();
        if (i >= inputTypes.size() || inputTypes.get(i).getDataClass() != java.sql.Date.class) {
            return null;
        }
        RexLiteral lit = (RexLiteral) operands.get(1);
        if (lit.getType().getSqlTypeName() != SqlTypeName.CHAR) {
            return null;
        }
        if (lit.getValue3() == null) {
            return col(i).binary(op, nullOf(GpuNative.T_INT64));
        }
        Object date = DataTypes.DateType.convertFrom(lit.getValueAs(String.class));
        if (!(date instanceof OriginalDate)) {
            return null;
        }
        return col(i).binary(op, lit(TimeStorage.writeDate(((OriginalDate) date).getMysqlDateTime())));
    }

    private static GpuExpression unaryOf(List<RexNode> operands, List<DataType> inputTypes, int op) {
        if (operands.size() != 1) {
            return null;
        }
        GpuExpression x = translate(operands.get(0), inputTypes);
        return x == null ? null : x.unary(op);
    }
}
