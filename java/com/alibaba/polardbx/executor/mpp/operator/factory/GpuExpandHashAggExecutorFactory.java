/*
 * GPU twin of HashAggExecutorFactory over the ExpandExec under it (mpp/operator/factory/HashAggExecutorFactory.java:49-106,
 * ExpandExecutorFactory): the HashAgg's constructor arguments plus the LogicalExpand, whose input feeds the executors
 * directly; selected in LocalExecutionPlanner.visitHashAgg when GpuSupport.groupingSetsSupported(...) holds and the agg is
 * partial or the pipeline's parallelism is 1 (INTEGRATION.md).
 */
package com.alibaba.polardbx.executor.mpp.operator.factory;

import com.alibaba.polardbx.executor.operator.Executor;
import com.alibaba.polardbx.executor.operator.GpuExpandHashAggExec;
import com.alibaba.polardbx.executor.operator.gpu.GpuAggSpec;
import com.alibaba.polardbx.executor.operator.gpu.GpuSupport;
import com.alibaba.polardbx.executor.utils.RuntimeStatHelper;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.alibaba.polardbx.optimizer.core.rel.HashAgg;
import com.alibaba.polardbx.optimizer.utils.CalciteUtils;
import org.apache.calcite.rel.logical.LogicalExpand;

import java.util.ArrayList;
import java.util.List;

public class GpuExpandHashAggExecutorFactory extends ExecutorFactory {
    private static final int MIN_HASH_TABLE_SIZE = 1024, MAX_HASH_TABLE_SIZE = 131064; // HashAggExecutorFactory.java:76-84

    private final HashAgg hashAgg;
    private final LogicalExpand expand;
    private final int parallelism, taskNumber;
    private final Integer rowCount;
    private final List<DataType> inputDataTypes; // the Expand's input
    private final List<Executor> executors = new ArrayList<>();

    public GpuExpandHashAggExecutorFactory(HashAgg hashAgg, LogicalExpand expand, int parallelism, int taskNumber,
                                           Integer rowCount, List<DataType> inputDataTypes) {
        this.hashAgg = hashAgg;
        this.expand = expand;
        this.parallelism = parallelism;
        this.taskNumber = taskNumber;
        this.rowCount = rowCount;
        this.inputDataTypes = inputDataTypes;
    }

    @Override
    public Executor createExecutor(ExecutionContext context, int index) {
        return createAllExecutors(context).get(index);
    }

    @Override
    public List<Executor> getAllExecutors(ExecutionContext context) {
        return createAllExecutors(context);
    }

    private synchronized List<Executor> createAllExecutors(ExecutionContext context) {
        if (executors.isEmpty()) {
            int[] groups = HashAggExecutorFactory.convertFrom(hashAgg.getGroupSet());
            int expected = rowCount == null ? MIN_HASH_TABLE_SIZE : rowCount / (taskNumber * parallelism);
            expected = Math.max(MIN_HASH_TABLE_SIZE, Math.min(MAX_HASH_TABLE_SIZE, expected));
            List<DataType> expandDataTypes = CalciteUtils.getTypes(expand.getRowType());
            GpuAggSpec spec = GpuAggSpec.tryConvert(hashAgg.getAggCallList(), expandDataTypes); // non-null: GpuSupport
            GpuSupport.ExpandItems items = GpuSupport.expandItems(expand);                      // non-null: GpuSupport
            List<DataType> outputDataTypes = CalciteUtils.getTypes(hashAgg.getRowType());
            for (int j = 0; j < parallelism; j++) {
                GpuExpandHashAggExec exec = new GpuExpandHashAggExec(inputDataTypes, items.src, items.col, items.value,
                    expandDataTypes, groups, spec, outputDataTypes, expected, context);
                exec.setId(hashAgg.getRelatedId());
                if (context.getRuntimeStatistics() != null) {
                    RuntimeStatHelper.registerStatForExec(hashAgg, exec, context);
                }
                executors.add(exec);
            }
        }
        return executors;
    }
}
