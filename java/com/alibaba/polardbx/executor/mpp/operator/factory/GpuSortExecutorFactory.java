/*
 * GPU twin of SortExecutorFactory (mpp/operator/factory/SortExecutorFactory.java): same constructor arguments (minus the
 * spiller: the GPU path does not spill) and the same OrderByOption conversion; selected in
 * LocalExecutionPlanner.visitMemSort when GpuSupport.sortSupported(...) holds.
 */
package com.alibaba.polardbx.executor.mpp.operator.factory;

import com.alibaba.polardbx.executor.operator.Executor;
import com.alibaba.polardbx.executor.operator.GpuSortExec;
import com.alibaba.polardbx.executor.utils.ExecUtils;
import com.alibaba.polardbx.executor.utils.OrderByOption;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.alibaba.polardbx.optimizer.core.rel.MemSort;
import com.alibaba.polardbx.statistics.RuntimeStatHelper;
import org.apache.calcite.rel.RelFieldCollation;

import java.util.ArrayList;
import java.util.List;

public class GpuSortExecutorFactory extends ExecutorFactory {
    private final MemSort sort;
    private final int parallelism;
    private final List<DataType> dataTypeList;
    private final List<Executor> executors = new ArrayList<>();

    public GpuSortExecutorFactory(MemSort sort, int parallelism, List<DataType> dataTypeList) {
        this.sort = sort;
        this.parallelism = parallelism;
        this.dataTypeList = dataTypeList;
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
            for (int j = 0; j < parallelism; j++) {
                List<RelFieldCollation> sortList = sort.getCollation().getFieldCollations();
                List<OrderByOption> orderBys = ExecUtils.convertFrom(sortList);
                GpuSortExec exec = new GpuSortExec(dataTypeList, orderBys, context);
                exec.setId(sort.getRelatedId());
                if (context.getRuntimeStatistics() != null) {
                    RuntimeStatHelper.registerStatForExec(sort, exec, context);
                }
                executors.add(exec);
            }
        }
        return executors;
    }
}
