/*
 * A scalar expression as the postfix program gsql_scan_* evaluates (include/gsql_gpu.h: gsql_expr, gsql_expr_op): the
 * GPU-side stand-in for a VectorizedExpression tree (executor/vectorized/**).  Programs are immutable; the builder
 * methods return new programs.  fromRex() translates the RexNode the planner hands to VectorizedExpressionBuilder and
 * returns null for anything the GPU path does not evaluate (the factory then keeps the stock operator).
 */
package com.alibaba.polardbx.executor.operator.gpu;

import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import org.apache.calcite.rex.RexCall;
import org.apache.calcite.rex.RexInputRef;
import org.apache.calcite.rex.RexLiteral;
import org.apache.calcite.rex.RexNode;

import java.math.BigDecimal;
import java.util.List;

public final class GpuExpression {
    // gsql_expr_op
    public static final int OP_COL = 1, OP_CONST_I64 = 2, OP_CONST_F64 = 3, OP_ADD = 4, OP_SUB = 5, OP_MUL = 6, OP_DIV = 7, OP_NEG = 8,
        OP_LT = 9, OP_LE = 10, OP_GT = 11, OP_GE = 12, OP_EQ = 13, OP_NE = 14, OP_AND = 15, OP_OR = 16, OP_NOT = 17, OP_IS_NULL = 18,
        OP_CAST_F64 = 19, OP_CAST_I64 = 20;
    /** GSQL_MAX_EXPR_INS */
    public static final int MAX_INSTRUCTIONS = 24;

    public final int[] ops;
    public final int[] args;
    /** constants: the long value, or Double.doubleToRawLongBits for OP_CONST_F64 */
    public final long[] consts;

    private GpuExpression(int[] ops, int[] args, long[] consts) {
        this.ops = ops;
        this.args = args;
        this.consts = consts;
    }

    private static GpuExpression one(int op, int arg, long k) {
        return new GpuExpression(new int[] {op}, new int[] {arg}, new long[] {k});
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

    private GpuExpression then(GpuExpression other, int op) {
        int n = ops.length + (other == null ? 0 : other.ops.length) + 1;
        int[] o = new int[n];
        int[] a = new int[n];
        long[] k = new long[n];
        System.arraycopy(ops, 0, o, 0, ops.length);
        System.arraycopy(args, 0, a, 0, ops.length);
        System.arraycopy(consts, 0, k, 0, ops.length);
        if (other != null) {
            System.arraycopy(other.ops, 0, o, ops.length, other.ops.length);
            System.arraycopy(other.args, 0, a, ops.length, other.ops.length);
            System.arraycopy(other.consts, 0, k, ops.length, other.ops.length);
        }
        o[n - 1] = op;
        return new GpuExpression(o, a, k);
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
     * RexNode -> program.  Covered: input refs over INT / BIGINT / DOUBLE columns, exact and approximate numeric
     * literals, + - * unary minus, `/` where the planner typed the quotient DOUBLE, the six comparisons, AND / OR / NOT,
     * IS NULL / IS NOT NULL, CAST to BIGINT / SIGNED / DOUBLE.
     */
    public static GpuExpression fromRex(RexNode node, List<DataType> inputTypes) {
        if (node instanceof RexInputRef) { // a bare column passes through whatever its block type (DATE / DATETIME as packed longs)
            int i = ((RexInputRef) node).getIndex();
            return i < inputTypes.size() && GpuTypes.code(inputTypes.get(i)) >= 0 ? col(i) : null;
        }
        GpuExpression e = translate(node, inputTypes);
        return e != null && e.fits() ? e : null;
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

    private static GpuExpression unaryOf(List<RexNode> operands, List<DataType> inputTypes, int op) {
        if (operands.size() != 1) {
            return null;
        }
        GpuExpression x = translate(operands.get(0), inputTypes);
        return x == null ? null : x.unary(op);
    }
}
