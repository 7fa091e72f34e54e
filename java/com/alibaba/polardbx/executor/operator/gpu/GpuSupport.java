package com.alibaba.polardbx.executor.operator.gpu;

import com.alibaba.polardbx.common.properties.ConnectionParams;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.alibaba.polardbx.optimizer.core.join.EquiJoinKey;
import com.alibaba.polardbx.optimizer.core.rel.HashAgg;
import com.alibaba.polardbx.optimizer.core.rel.SortAgg;
import com.alibaba.polardbx.optimizer.core.rel.SortWindow;
import com.alibaba.polardbx.optimizer.utils.CalciteUtils;
import org.apache.calcite.rel.RelFieldCollation;
import org.apache.calcite.rel.core.AggregateCall;
import org.apache.calcite.rel.core.Join;
import org.apache.calcite.rel.core.JoinRelType;
import org.apache.calcite.rel.core.Window;
import org.apache.calcite.rel.logical.LogicalExpand;
import org.apache.calcite.rel.type.RelDataType;
import org.apache.calcite.rex.RexInputRef;
import org.apache.calcite.rex.RexLiteral;
import org.apache.calcite.rex.RexNode;
import org.apache.calcite.sql.SqlKind;
import org.apache.calcite.sql.type.SqlTypeName;
import org.apache.calcite.util.ImmutableBitSet;

import java.util.ArrayList;
import java.util.List;

/**
 * Planner-time decisions (LocalExecutionPlanner.visitHashJoin:852 / visitHashAgg:1487): a GPU factory is chosen only
 * when the whole operator can run on the device; otherwise the stock factory is used.  There is no CPU fallback
 * inside a GPU operator.
 */
public final class GpuSupport {
    private GpuSupport() {
    }

    public static boolean enabled(ExecutionContext context) {
        return context.getParamManager().getBoolean(ConnectionParams.ENABLE_GPU_OPERATORS) && GpuDevices.count() > 0;
    }

    public static boolean joinSupported(Join join, List<EquiJoinKey> keys, RexNode otherCond, boolean maxOneRow,
                                        List<RexNode> antiOperands, ExecutionContext context) {
        if (!enabled(context)) {
            return false;
        }
        JoinRelType t = join.getJoinType();
        if (GpuTypes.joinType(t) < 0 || keys.isEmpty() || keys.size() > 8) {
            return false;
        }
        if ((t == JoinRelType.SEMI || t == JoinRelType.ANTI) && maxOneRow) {
            return false; // single semi/anti joins: GSQL_E_UNSUPPORTED at create
        }
        if (!GpuTypes.supported(CalciteUtils.getTypes(join.getOuter().getRowType()))
            || !GpuTypes.supported(CalciteUtils.getTypes(join.getInner().getRowType()))) {
            return false;
        }
        for (EquiJoinKey k : keys) {
            if (GpuTypes.code(k.getUnifiedType()) < 0 || k.isNullSafeEqual()) {
                return false;
            }
        }
        if (antiOperands != null) {
            for (RexNode o : antiOperands) {
                if (!(o instanceof org.apache.calcite.rex.RexInputRef)) {
                    return false; // NOT IN over expressions: stock operator
                }
            }
        }
        return GpuJoinCondition.convertible(otherCond);
    }

    /**
     * SortMergeJoinExec (SortMergeJoinFactory): joinSupported's type, key-count, null-safe-key and anti-operand checks, and
     * what gsql_smj refuses besides: any other condition (the stock operator emits a NULL-padded row for an outer row whose
     * last run row fails the condition even when earlier rows matched, and the GPU operator does not restate that), and
     * max-one-row semi, anti and right joins.
     */
    public static boolean sortMergeJoinSupported(Join join, List<EquiJoinKey> keys, RexNode otherCond, boolean maxOneRow,
                                                 List<RexNode> antiOperands, ExecutionContext context) {
        if (otherCond != null || (maxOneRow && join.getJoinType() == JoinRelType.RIGHT)) {
            return false;
        }
        return joinSupported(join, keys, null, maxOneRow, antiOperands, context);
    }

    /**
     * Runtime filters (RuntimeFilterBuilderExec on the build side, FilterExec with BLOOMFILTER(key) calls on the probe
     * side): the GPU builds and tests the xxhash_64 method only (ENABLE_RUNTIME_FILTER_XXHASH, the default), one key column
     * per filter (JoinToRuntimeFilterJoinRule.java:157-214 never emits more), keys INT / BIGINT / DOUBLE or DATE / DATETIME
     * (packed longs, hashed with putLong like LongBlock: DateBlock.java:146-152), every column a type GpuChunks stages.
     * Otherwise the stock operator runs.
     */
    public static boolean runtimeFilterSupported(List<DataType> inputTypes, List<List<Integer>> keys, ExecutionContext context) {
        if (!enabled(context) || !context.getParamManager().getBoolean(ConnectionParams.ENABLE_RUNTIME_FILTER_XXHASH)) {
            return false;
        }
        if (keys.isEmpty() || !GpuTypes.supported(inputTypes)) {
            return false;
        }
        for (List<Integer> k : keys) {
            if (k.size() != 1 || GpuTypes.code(inputTypes.get(k.get(0))) < 0) {
                return false;
            }
        }
        return true;
    }

    /** gsql_sort_spec holds at most GSQL_MAX_KEYS sort keys and GSQL_MAX_COLS columns (include/gsql_gpu.h). */
    static final int MAX_SORT_KEYS = 8, MAX_SORT_COLS = 32;

    /**
     * MemSort (SortExec) and TopN (SpilledTopNExec): the GPU orders INT / BIGINT / DOUBLE columns and DATE / DATETIME /
     * TIMESTAMP columns, which arrive as packed longs that DateType.compare and TimestampType.compare order by Long.compare
     * (DateBlock / TimestampBlock.getObjectForCmp return the packed long), i.e. as BIGINT.  Any other column type (DECIMAL,
     * CHAR, ...) anywhere in the row, more than GSQL_MAX_KEYS keys or more than GSQL_MAX_COLS columns keep the stock
     * operator.  The collations' null direction needs no check: ExecUtils.getComparator never reads it.
     */
    public static boolean sortSupported(List<DataType> inputTypes, List<RelFieldCollation> collations, ExecutionContext context) {
        if (!enabled(context) || collations.isEmpty() || collations.size() > MAX_SORT_KEYS || inputTypes.size() > MAX_SORT_COLS) {
            return false;
        }
        if (!GpuTypes.supported(inputTypes)) {
            return false;
        }
        for (RelFieldCollation c : collations) {
            int i = c.getFieldIndex();
            if (i < 0 || i >= inputTypes.size()) {
                return false;
            }
        }
        return true;
    }

    /** GSQL_MAX_MERGE_INPUTS (include/gsql_gpu.h): the most runs one gsql_merge takes. */
    static final int MAX_MERGE_INPUTS = 4096;

    /**
     * MergeSortExec (LocalMergeSortExecutorFactory): the bounds of sortSupported (the merge orders rows with the same
     * comparator and spec), plus at most GSQL_MAX_MERGE_INPUTS inputs.
     */
    public static boolean mergeSortSupported(List<DataType> inputTypes, List<RelFieldCollation> collations, int childParallelism,
                                             ExecutionContext context) {
        if (childParallelism < 1 || childParallelism > MAX_MERGE_INPUTS) {
            return false;
        }
        return sortSupported(inputTypes, collations, context);
    }

    public static boolean aggSupported(HashAgg agg, List<DataType> inputTypes, ExecutionContext context) {
        return aggShapeSupported(agg.getGroupSet(), agg.getRowType(), agg.getAggCallList(), inputTypes, context);
    }

    /**
     * SortWindow through NonFrameOverWindowExec (OverWindowFramesExecFactory.java:78-87,136-164): only when the first call
     * of groups.get(0) is ROW_NUMBER, RANK or DENSE_RANK (the factory's own selection) and the window has that one group
     * (the stock operator computes group 0's calls only).  Every call must convert (GpuAggSpec.tryConvertWindow: no FILTER,
     * no DISTINCT, at most 4 RANK columns), partition keys and outputs must be INT / BIGINT / DOUBLE (DATE as its packed
     * BIGINT): DECIMAL anywhere keeps the stock operator.  The types come from the plan, so the decision is made before
     * any child executor exists.
     * The stock factory picks each aggregator's class from dataTypes.subList(groups.length, ...) (:147-150): the type of
     * the window's column npart + i, not of call i's output column nInput + i.  Where the two differ the stock aggregator
     * is not the one the call's type names (e.g. the generic Sum for SUM(DOUBLE) over a BIGINT slot), so an aggregate call
     * is refused unless they agree; the rank family ignores the type.
     */
    public static boolean nonFrameWindowSupported(SortWindow window, ExecutionContext context) {
        if (!enabled(context) || window.groups.size() != 1) {
            return false;
        }
        Window.Group group = window.groups.get(0);
        SqlKind first = group.aggCalls.get(0).getOperator().getKind();
        if (first != SqlKind.ROW_NUMBER && first != SqlKind.RANK && first != SqlKind.DENSE_RANK) {
            return false;
        }
        List<DataType> inputTypes = CalciteUtils.getTypes(window.getInput().getRowType());
        List<DataType> dataTypes = CalciteUtils.getTypes(window.getRowType());
        if (group.keys.cardinality() > 8 || !GpuTypes.supported(inputTypes) || !GpuTypes.supported(dataTypes)) {
            return false;
        }
        List<AggregateCall> calls = group.getAggregateCalls(window);
        GpuAggSpec spec = GpuAggSpec.tryConvertWindow(calls, inputTypes);
        if (spec == null || spec.producesDecimal(inputTypes)) {
            return false;
        }
        int npart = group.keys.cardinality();
        for (int i = 0; i < calls.size(); i++) {
            boolean rankFamily = spec.kinds[i] == GpuAggSpec.ROW_NUMBER || spec.kinds[i] == GpuAggSpec.RANK
                || spec.kinds[i] == GpuAggSpec.DENSE_RANK;
            DataType stockType = dataTypes.get(npart + i);                  // what the stock factory passes
            DataType callType = dataTypes.get(inputTypes.size() + i);      // the call's output column
            if (!rankFamily && (stockType.getDataClass() != callType.getDataClass()
                || GpuTypes.code(stockType) != GpuTypes.code(callType))) {
                return false;
            }
        }
        return true;
    }

    /**
     * SortAggExec (SortAggExecFactory): aggSupported's checks, and no FILTER argument.  The stock SortAggExec ignores a
     * FILTER clause (it calls Aggregator.accumulate directly); gsql_sortagg refuses one rather than diverge, so such plans
     * keep the stock operator.  Calls GpuAggSpec does not know (e.g. GROUP_CONCAT, DISTINCT) make tryConvert return null;
     * __FIRST_VALUE is known, and refused with a FILTER argument on both aggregations.
     */
    public static boolean sortAggSupported(SortAgg agg, List<DataType> inputTypes, ExecutionContext context) {
        for (AggregateCall call : agg.getAggCallList()) {
            if (call.filterArg >= 0) {
                return false;
            }
        }
        return aggShapeSupported(agg.getGroupSet(), agg.getRowType(), agg.getAggCallList(), inputTypes, context);
    }

    /** GSQL_MAX_SETS (include/gsql_gpu.h): the most grouping sets one gsql_gsagg takes (CUBE of four keys). */
    static final int MAX_SETS = 16;

    /** An Expand's projections as gsql_expand_item fields: src[s][c] (GpuNative.EXPAND_*), col[s][c], value[s][c]. */
    public static final class ExpandItems {
        public final int[][] src, col;
        public final long[][] value;

        ExpandItems(int nsets, int ncols) {
            src = new int[nsets][ncols];
            col = new int[nsets][ncols];
            value = new long[nsets][ncols];
        }
    }

    /**
     * The projections of a LogicalExpand (GroupingSetsToExpandRule.java:255-300) as the device takes them: every item a
     * RexInputRef, a NULL literal or an exact integer literal; anything else (null) keeps the stock ExpandExec.
     */
    public static ExpandItems expandItems(LogicalExpand expand) {
        List<List<RexNode>> projects = expand.getProjects();
        if (projects.isEmpty()) {
            return null;
        }
        ExpandItems it = new ExpandItems(projects.size(), projects.get(0).size());
        for (int s = 0; s < projects.size(); s++) {
            List<RexNode> p = projects.get(s);
            for (int c = 0; c < p.size(); c++) {
                RexNode n = p.get(c);
                if (n instanceof RexInputRef) {
                    it.src[s][c] = GpuNative.EXPAND_INPUT;
                    it.col[s][c] = ((RexInputRef) n).getIndex();
                } else if (RexLiteral.isNullLiteral(n)) {
                    it.src[s][c] = GpuNative.EXPAND_NULL;
                } else if (n instanceof RexLiteral && SqlTypeName.INT_TYPES.contains(n.getType().getSqlTypeName())
                    && ((RexLiteral) n).getValue2() instanceof Number) {
                    it.src[s][c] = GpuNative.EXPAND_CONST;
                    it.value[s][c] = ((Number) ((RexLiteral) n).getValue2()).longValue();
                } else {
                    return null;
                }
            }
        }
        return it;
    }

    /**
     * HashAgg over LogicalExpand (ROLLUP / CUBE / GROUPING SETS and the DISTINCT rewrites) as one gsql_gsagg: aggSupported's
     * checks over the Expand's output, expandItems' item forms, and gsql_gsagg_create's refusals — no __FIRST_VALUE (its
     * first-row and one-group rules span the whole aggregation); every aggregate argument and FILTER column a reference to
     * the same input column in every set; a reference only where the input column has the output column's type (else the
     * stock DataTypeUtils.convert would change the value); constants only in INT / BIGINT columns, within INT range in an
     * INT column; a group column holding pairwise distinct constants in all sets ($e, GroupingSetsToExpandRule's
     * genExpandId), without which groups of different sets could coincide; 1..GSQL_MAX_SETS sets.
     * The caller also requires agg.isPartial() or a pipeline parallelism of 1 (INTEGRATION.md, visitHashAgg): otherwise the
     * local exchange partitions the expanded rows by (keys, $e), which the unexpanded rows cannot be routed by.
     */
    public static boolean groupingSetsSupported(HashAgg agg, LogicalExpand expand, List<DataType> inputTypes,
                                                ExecutionContext context) {
        ExpandItems it = expandItems(expand);
        if (it == null || it.src.length < 1 || it.src.length > MAX_SETS || !GpuTypes.supported(inputTypes)) {
            return false;
        }
        List<DataType> outTypes = CalciteUtils.getTypes(expand.getRowType());
        if (!aggShapeSupported(agg.getGroupSet(), agg.getRowType(), agg.getAggCallList(), outTypes, context)) {
            return false;
        }
        int nsets = it.src.length;
        for (int s = 0; s < nsets; s++) {
            for (int c = 0; c < outTypes.size(); c++) {
                int code = GpuTypes.code(outTypes.get(c));
                if (it.src[s][c] == GpuNative.EXPAND_INPUT) {
                    DataType in = inputTypes.get(it.col[s][c]);
                    if (GpuTypes.code(in) != code || in.getDataClass() != outTypes.get(c).getDataClass()) {
                        return false;
                    }
                } else if (it.src[s][c] == GpuNative.EXPAND_CONST) {
                    long v = it.value[s][c];
                    if (code == GpuNative.T_FP64 || (code == GpuNative.T_INT32 && (v < Integer.MIN_VALUE || v > Integer.MAX_VALUE))) {
                        return false;
                    }
                }
            }
        }
        for (AggregateCall call : agg.getAggCallList()) {
            if (call.getAggregation().getKind() == SqlKind.__FIRST_VALUE) {
                return false;
            }
            List<Integer> used = new ArrayList<>(call.getArgList());
            if (call.filterArg >= 0) {
                used.add(call.filterArg);
            }
            for (int c : used) {
                for (int s = 0; s < nsets; s++) {
                    if (it.src[s][c] != GpuNative.EXPAND_INPUT || it.col[s][c] != it.col[0][c]) {
                        return false;
                    }
                }
            }
        }
        for (int g : agg.getGroupSet()) {
            boolean distinct = true;
            for (int s = 0; s < nsets && distinct; s++) {
                distinct = it.src[s][g] == GpuNative.EXPAND_CONST;
                for (int q = 0; q < s && distinct; q++) {
                    distinct = it.value[q][g] != it.value[s][g];
                }
            }
            if (distinct) {
                return true;
            }
        }
        return false;
    }

    private static boolean aggShapeSupported(ImmutableBitSet groupSet, RelDataType rowType, List<AggregateCall> calls,
                                             List<DataType> inputTypes, ExecutionContext context) {
        if (!enabled(context) || groupSet.cardinality() > 8) {
            return false;
        }
        if (!GpuTypes.supported(CalciteUtils.getTypes(rowType))) {
            return false; // e.g. SUM(BIGINT) -> DECIMAL output
        }
        // every input column crosses to the device (GpuTypes.codes in GpuHashAggExec / GpuSortAggExec throws on any column
        // without a GPU type, including a FILTER column or one no call reads): such plans keep the stock operator
        if (!GpuTypes.supported(inputTypes)) {
            return false;
        }
        for (int g : groupSet) {
            if (GpuTypes.code(inputTypes.get(g)) < 0) {
                return false;
            }
        }
        GpuAggSpec spec = GpuAggSpec.tryConvert(calls, inputTypes);
        return spec != null && !spec.producesDecimal(inputTypes);
    }
}
