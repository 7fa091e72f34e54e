/*
 * GPU twin of OverWindowFramesExecFactory (mpp/operator/factory/OverWindowFramesExecFactory.java) for the operator it builds
 * for rank-family windows, NonFrameOverWindowExec.  Same constructor; when GpuSupport.nonFrameWindowSupported(...) holds it
 * builds GpuNonFrameOverWindowExec with the calls, partition keys and CURRENT ROW .. CURRENT ROW flag the stock factory
 * would pass (:136-164), and otherwise defers to super, which builds the stock NonFrameOverWindowExec or
 * OverWindowFramesExec.  The choice is made from the plan alone, before any child executor is created, so each branch
 * creates its child exactly once (a LogicalView child registers every TableScanExec it builds with its scan client).
 * Selected in LocalExecutionPlanner.createOverWindowFactory (INTEGRATION.md).
 */
package com.alibaba.polardbx.executor.mpp.operator.factory;

import com.alibaba.polardbx.executor.operator.Executor;
import com.alibaba.polardbx.executor.operator.GpuNonFrameOverWindowExec;
import com.alibaba.polardbx.executor.operator.gpu.GpuAggSpec;
import com.alibaba.polardbx.executor.operator.gpu.GpuSupport;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.alibaba.polardbx.optimizer.core.rel.SortWindow;
import com.alibaba.polardbx.optimizer.utils.CalciteUtils;
import com.alibaba.polardbx.statistics.RuntimeStatHelper;
import org.apache.calcite.rel.core.Window;

import java.util.List;

public class GpuNonFrameOverWindowExecFactory extends OverWindowFramesExecFactory {
    private final SortWindow overWindow;

    public GpuNonFrameOverWindowExecFactory(SortWindow overWindow, ExecutorFactory executorFactory) {
        super(overWindow, executorFactory);
        this.overWindow = overWindow;
    }

    @Override
    public Executor createExecutor(ExecutionContext context, int index) {
        if (!GpuSupport.nonFrameWindowSupported(overWindow, context)) {
            return super.createExecutor(context, index);
        }
        Executor input = getInputs().get(0).createExecutor(context, index);
        Window.Group group = overWindow.groups.get(0);
        List<DataType> dataTypes = CalciteUtils.getTypes(overWindow.getRowType());
        GpuAggSpec spec = GpuAggSpec.tryConvertWindow(group.getAggregateCalls(overWindow), input.getDataTypes());
        boolean reset = group.lowerBound.isCurrentRow() && group.upperBound.isCurrentRow();
        Executor exec = new GpuNonFrameOverWindowExec(input, context, spec, group.keys.asList(), reset, dataTypes);
        exec.setId(overWindow.getRelatedId());
        if (context.getRuntimeStatistics() != null) {
            RuntimeStatHelper.registerStatForExec(overWindow, exec, context);
        }
        return exec;
    }
}
