/*
 * GPU twin of SortAggExecFactory (mpp/operator/factory/SortAggExecFactory.java): same constructor, one executor per
 * driver over the child factory's executor of that driver, the same AggregateUtils.convertAggregators output types.
 * When GpuSupport.sortAggSupported(...) is false it builds the stock SortAggExec instead; selected in
 * LocalExecutionPlanner.visitSortAgg (INTEGRATION.md).
 */
package com.alibaba.polardbx.executor.mpp.operator.factory;

import com.alibaba.polardbx.executor.calc.Aggregator;
import com.alibaba.polardbx.executor.operator.Executor;
import com.alibaba.polardbx.executor.operator.GpuSortAggExec;
import com.alibaba.polardbx.executor.operator.SortAggExec;
import com.alibaba.polardbx.executor.operator.gpu.GpuAggSpec;
import com.alibaba.polardbx.executor.operator.gpu.GpuSupport;
import com.alibaba.polardbx.executor.operator.util.AggregateUtils;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.alibaba.polardbx.optimizer.core.rel.SortAgg;
import com.alibaba.polardbx.optimizer.memory.MemoryAllocatorCtx;
import com.alibaba.polardbx.optimizer.utils.CalciteUtils;
import com.alibaba.polardbx.statistics.RuntimeStatHelper;

import java.util.ArrayList;
import java.util.List;

import static com.alibaba.polardbx.executor.mpp.operator.factory.HashAggExecutorFactory.convertFrom;

public class GpuSortAggExecFactory extends ExecutorFactory {
    private final SortAgg sortAgg;
    private final int parallelism;
    private final List<Executor> executors = new ArrayList<>();

    public GpuSortAggExecFactory(SortAgg sortAgg, ExecutorFactory executorFactory, int parallelism) {
        this.sortAgg = sortAgg;
        this.parallelism = parallelism;
        addInput(executorFactory);
    }

    @Override
    public Executor createExecutor(ExecutionContext context, int index) {
        getAllExecutors(context);
        return executors.get(index);
    }

    @Override
    public synchronized List<Executor> getAllExecutors(ExecutionContext context) {
        if (executors.isEmpty()) {
            for (int k = 0; k < parallelism; k++) {
                Executor input = getInputs().get(0).createExecutor(context, k);
                List<DataType> outputDataTypes = CalciteUtils.getTypes(sortAgg.getRowType());
                int[] groups = convertFrom(sortAgg.getGroupSet());
                Executor exec;
                if (GpuSupport.sortAggSupported(sortAgg, input.getDataTypes(), context)) {
                    GpuAggSpec spec = GpuAggSpec.tryConvert(sortAgg.getAggCallList(), input.getDataTypes());
                    exec = new GpuSortAggExec(input, groups, spec, outputDataTypes, context);
                } else {
                    MemoryAllocatorCtx memoryAllocator = context.getMemoryPool().getMemoryAllocatorCtx();
                    List<Aggregator> aggregators = AggregateUtils.convertAggregators(input.getDataTypes(),
                        outputDataTypes.subList(sortAgg.getGroupCount(), sortAgg.getGroupCount() + sortAgg.getAggCallList().size()),
                        sortAgg.getAggCallList(), context, memoryAllocator);
                    exec = new SortAggExec(input, groups, aggregators, outputDataTypes, context);
                }
                exec.setId(sortAgg.getRelatedId());
                if (context.getRuntimeStatistics() != null) {
                    RuntimeStatHelper.registerStatForExec(sortAgg, exec, context);
                }
                executors.add(exec);
            }
        }
        return executors;
    }
}
