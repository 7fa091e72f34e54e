/*
 * GPU twin of SortMergeJoinFactory (mpp/operator/factory/SortMergeJoinFactory.java): same constructor, one executor per
 * index over the inner and outer factories' executors of that index (the two sides' partitions are aligned), the same
 * EquiJoinKeys and anti-join operands.  When GpuSupport.sortMergeJoinSupported(...) is false it builds the stock
 * SortMergeJoinExec instead; selected in LocalExecutionPlanner.visitSortMergeJoin (INTEGRATION.md).
 */
package com.alibaba.polardbx.executor.mpp.operator.factory;

import com.alibaba.polardbx.executor.operator.Executor;
import com.alibaba.polardbx.executor.operator.GpuSortMergeJoinExec;
import com.alibaba.polardbx.executor.operator.SortMergeJoinExec;
import com.alibaba.polardbx.executor.operator.gpu.GpuSupport;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.expression.calc.IExpression;
import com.alibaba.polardbx.optimizer.core.join.EquiJoinKey;
import com.alibaba.polardbx.optimizer.core.join.EquiJoinUtils;
import com.alibaba.polardbx.optimizer.utils.CalciteUtils;
import com.alibaba.polardbx.optimizer.utils.RexUtils;
import com.alibaba.polardbx.statistics.RuntimeStatHelper;
import org.apache.calcite.rel.core.Join;
import org.apache.calcite.rel.core.JoinRelType;
import org.apache.calcite.rex.RexInputRef;
import org.apache.calcite.rex.RexNode;

import java.util.ArrayList;
import java.util.List;
import java.util.stream.Collectors;

public class GpuSortMergeJoinFactory extends ExecutorFactory {
    private final Join join;
    private final List<Integer> leftColumns;
    private final List<Integer> rightColumns;
    private final List<Boolean> columnIsAscending;
    private final RexNode otherCond;
    private final List<RexNode> operands;
    private final boolean maxOneRow;

    public GpuSortMergeJoinFactory(Join join, List<Integer> leftColumns, List<Integer> rightColumns,
                                   List<Boolean> columnIsAscending, RexNode otherCond,
                                   List<RexNode> operands, boolean maxOneRow, ExecutorFactory inner, ExecutorFactory outer) {
        this.join = join;
        this.leftColumns = leftColumns;
        this.rightColumns = rightColumns;
        this.columnIsAscending = columnIsAscending;
        this.otherCond = otherCond;
        this.operands = operands;
        this.maxOneRow = maxOneRow;
        addInput(inner);
        addInput(outer);
    }

    @Override
    public Executor createExecutor(ExecutionContext context, int index) {
        Executor inner = getInputs().get(0).createExecutor(context, index);
        Executor outer = getInputs().get(1).createExecutor(context, index);
        JoinRelType joinType = join.getJoinType();
        List<EquiJoinKey> joinKeys = EquiJoinUtils.buildEquiJoinKeys(join.getOuter(), join.getInner(),
            joinType.outerSide(leftColumns, rightColumns), joinType.innerSide(leftColumns, rightColumns));
        boolean anti = operands != null && joinType == JoinRelType.ANTI && !operands.isEmpty();
        Executor ret;
        if (GpuSupport.sortMergeJoinSupported(join, joinKeys, otherCond, maxOneRow, anti ? operands : null, context)) {
            int[] antiOperands = anti ? operands.stream().mapToInt(o -> ((RexInputRef) o).getIndex()).toArray() : null;
            ret = new GpuSortMergeJoinExec(outer, inner, joinType, maxOneRow, joinKeys, columnIsAscending, antiOperands,
                CalciteUtils.getTypes(join.getRowType()), context);
        } else {
            IExpression otherCondition = convertExpression(otherCond, context);
            List<IExpression> antiJoinOperands = null;
            if (anti) {
                antiJoinOperands = operands.stream().map(e -> convertExpression(e, context)).collect(Collectors.toList());
            }
            ret = new SortMergeJoinExec(outer, inner, joinType, maxOneRow, joinKeys, columnIsAscending, otherCondition,
                antiJoinOperands, context);
        }
        ret.setId(join.getRelatedId());
        if (context.getRuntimeStatistics() != null) {
            RuntimeStatHelper.registerStatForExec(join, ret, context);
        }
        return ret;
    }

    private IExpression convertExpression(RexNode rexNode, ExecutionContext context) {
        return RexUtils.buildRexNode(rexNode, context, new ArrayList<>());
    }
}
