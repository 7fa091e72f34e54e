package com.alibaba.polardbx.executor.operator.gpu;

import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import org.apache.calcite.rel.core.AggregateCall;
import org.apache.calcite.sql.SqlKind;

import java.util.List;

/**
 * gsql_agg_call list derived from the plan's AggregateCalls, by the same case analysis as
 * AggregateUtils.convertAggregators (operator/util/AggregateUtils.java:120-330) — restricted to the aggregators the GPU
 * path restates (SURVEY §8a a10).  tryConvert returns null otherwise: planner-time fall-through, never a runtime one.
 */
public final class GpuAggSpec {
    public static final int COUNT_STAR = 0, COUNT = 1, SUM = 2, AVG = 3, MIN = 4, MAX = 5, SUM0 = 6, FIRST_VALUE = 8;
    public static final int ROW_NUMBER = 9, RANK = 10, DENSE_RANK = 11; // gsql_window only

    public final int[] kinds;
    public final int[][] cols;
    public final int[] filterArgs;

    private GpuAggSpec(int[] kinds, int[][] cols, int[] filterArgs) {
        this.kinds = kinds;
        this.cols = cols;
        this.filterArgs = filterArgs;
    }

    public static GpuAggSpec tryConvert(List<AggregateCall> calls, List<DataType> inputTypes) {
        int n = calls.size();
        if (n > 16) {
            return null; // GSQL_MAX_AGGS
        }
        int[] kinds = new int[n];
        int[][] cols = new int[n][];
        int[] filters = new int[n];
        for (int i = 0; i < n; i++) {
            AggregateCall call = calls.get(i);
            if (call.isDistinct()) {
                return null; // DISTINCT aggregates keep the stock operator (out of v1 scope)
            }
            List<Integer> args = call.getArgList();
            if (args.size() > 4) {
                return null;
            }
            cols[i] = new int[args.size()];
            for (int a = 0; a < args.size(); a++) {
                cols[i][a] = args.get(a);
                if (GpuTypes.code(inputTypes.get(args.get(a))) < 0) {
                    return null;
                }
            }
            // AggOpenHashMap.putChunk filters a row only on a Long cell below 1.  A DATE / DATETIME / TIMESTAMP filter column
            // reaches the GPU as its packed BIGINT, which the kernels would test as a Long, while the stock operator sees a
            // Date / Timestamp object and never filters: keep the stock operator for any filter column that is not numeric
            if (call.filterArg >= 0 && !GpuTypes.isNumeric(inputTypes.get(call.filterArg))) {
                return null;
            }
            filters[i] = call.filterArg;
            int arg0 = args.isEmpty() ? -1 : GpuTypes.code(inputTypes.get(args.get(0)));
            SqlKind kind = call.getAggregation().getKind();
            switch (kind) {
            case COUNT:
                kinds[i] = args.isEmpty() ? COUNT_STAR : COUNT;
                break;
            case SUM:
                if (args.size() != 1) {
                    return null;
                }
                kinds[i] = SUM; // DOUBLE -> DOUBLE (Double2DoubleSum); INT/BIGINT -> exact DECIMAL (Long2DecimalSum)
                break;
            case SUM0:
                if (args.size() != 1 || arg0 != GpuNative.T_INT64) {
                    return null;
                }
                kinds[i] = SUM0;
                break;
            case AVG:
                if (args.size() != 1 || arg0 != GpuNative.T_FP64) {
                    return null; // AVG over integers divides DECIMALs
                }
                kinds[i] = AVG;
                break;
            case MIN:
            case MAX:
                if (args.size() != 1) {
                    return null;
                }
                kinds[i] = kind == SqlKind.MIN ? MIN : MAX;
                break;
            case __FIRST_VALUE:
                // InternalFirstValue with a FILTER argument fails in the stock operator once a group's first row is
                // filtered out; gsql_agg_create refuses it, so such plans keep the stock operator
                if (args.size() != 1 || call.filterArg >= 0) {
                    return null;
                }
                kinds[i] = FIRST_VALUE; // INT / BIGINT / DOUBLE (DATE as a packed BIGINT) -> the same type
                break;
            default:
                return null;
            }
        }
        return new GpuAggSpec(kinds, cols, filters);
    }

    /**
     * The calls of a NonFrameOverWindowExec (AggregateUtils.convertWindowFunction for the rank family, convertAggregators
     * otherwise): ROW_NUMBER, RANK / DENSE_RANK over at most 4 INT / BIGINT / DOUBLE columns, and the aggregates tryConvert
     * accepts except __FIRST_VALUE.  Null for anything else, and for any FILTER argument (the stock operator ignores it).
     */
    public static GpuAggSpec tryConvertWindow(List<AggregateCall> calls, List<DataType> inputTypes) {
        int n = calls.size();
        if (n == 0 || n > 16) {
            return null;
        }
        int[] kinds = new int[n];
        int[][] cols = new int[n][];
        int[] filters = new int[n];
        for (int i = 0; i < n; i++) {
            AggregateCall call = calls.get(i);
            if (call.filterArg >= 0 || call.isDistinct()) {
                return null;
            }
            SqlKind kind = call.getAggregation().getKind();
            List<Integer> args = call.getArgList();
            if (kind == SqlKind.ROW_NUMBER || kind == SqlKind.RANK || kind == SqlKind.DENSE_RANK) {
                int[] a = kind == SqlKind.ROW_NUMBER || args.isEmpty() || args.get(0) < 0 ? new int[0]
                    : args.stream().mapToInt(Integer::intValue).toArray(); // Rank's constructor keeps index[0] >= 0 lists
                if (a.length > 4) {
                    return null;
                }
                for (int c : a) {
                    if (GpuTypes.code(inputTypes.get(c)) < 0) {
                        return null;
                    }
                }
                kinds[i] = kind == SqlKind.ROW_NUMBER ? ROW_NUMBER : kind == SqlKind.RANK ? RANK : DENSE_RANK;
                cols[i] = a;
                continue;
            }
            GpuAggSpec one = tryConvert(calls.subList(i, i + 1), inputTypes);
            if (one == null || one.kinds[0] == FIRST_VALUE) {
                return null;
            }
            kinds[i] = one.kinds[0];
            cols[i] = one.cols[0];
        }
        java.util.Arrays.fill(filters, -1);
        return new GpuAggSpec(kinds, cols, filters);
    }

    /** SUM over INT/BIGINT comes back as DEC128, which needs a DecimalBlock on the Java side: not produced yet. */
    public boolean producesDecimal(List<DataType> inputTypes) {
        for (int i = 0; i < kinds.length; i++) {
            if (kinds[i] == SUM && GpuTypes.code(inputTypes.get(cols[i][0])) != GpuNative.T_FP64) {
                return true;
            }
        }
        return false;
    }
}
