/*
 * GPU twin of LocalMergeSortExecutorFactory (mpp/operator/factory/LocalMergeSortExecutorFactory.java): same constructor
 * arguments and the same offset / limit extraction (limit Long.MAX_VALUE and offset 0 unless the Sort has a fetch).
 * Builds GpuMergeSortExec over the child's childParallelism executors when GpuSupport.mergeSortSupported(...) holds for
 * the row types, and the stock MergeSortExec otherwise; selected in LocalExecutionPlanner where the local merge-sort
 * factory is built (INTEGRATION.md).
 */
package com.alibaba.polardbx.executor.mpp.operator.factory;

import com.alibaba.polardbx.common.jdbc.ParameterContext;
import com.alibaba.polardbx.executor.operator.Executor;
import com.alibaba.polardbx.executor.operator.GpuMergeSortExec;
import com.alibaba.polardbx.executor.operator.MergeSortExec;
import com.alibaba.polardbx.executor.operator.gpu.GpuSupport;
import com.alibaba.polardbx.executor.utils.ExecUtils;
import com.alibaba.polardbx.executor.utils.OrderByOption;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.statistics.RuntimeStatHelper;
import org.apache.calcite.rel.RelFieldCollation;
import org.apache.calcite.rel.core.Sort;

import java.util.ArrayList;
import java.util.List;
import java.util.Map;

import static com.alibaba.polardbx.optimizer.core.planner.rule.util.CBOUtil.getRexParam;

public class GpuLocalMergeSortExecutorFactory extends ExecutorFactory {
    private final Sort sort;
    private final int childParallelism;
    private final List<Executor> executors = new ArrayList<>();

    public GpuLocalMergeSortExecutorFactory(Sort sort, ExecutorFactory executorFactory, int childParallelism) {
        this.sort = sort;
        this.childParallelism = childParallelism;
        addInput(executorFactory);
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
            List<Executor> inputs = new ArrayList<>();
            for (int i = 0; i < childParallelism; i++) {
                inputs.add(getInputs().get(0).createExecutor(context, i));
            }
            List<RelFieldCollation> sortList = sort.getCollation().getFieldCollations();
            List<OrderByOption> orderBys = ExecUtils.convertFrom(sortList);
            long limit = Long.MAX_VALUE;
            long offset = 0;
            Map<Integer, ParameterContext> params = context.getParams().getCurrentParameter();
            if (sort.fetch != null) {
                limit = getRexParam(sort.fetch, params);
                if (sort.offset != null) {
                    offset = getRexParam(sort.offset, params);
                }
            }
            Executor exec;
            if (GpuSupport.mergeSortSupported(inputs.get(0).getDataTypes(), sortList, childParallelism, context)) {
                exec = new GpuMergeSortExec(inputs, orderBys, offset, limit, context);
            } else {
                exec = new MergeSortExec(inputs, orderBys, offset, limit, context);
            }
            exec.setId(sort.getRelatedId());
            if (context.getRuntimeStatistics() != null) {
                RuntimeStatHelper.registerStatForExec(sort, exec, context);
            }
            executors.add(exec);
        }
        return executors;
    }
}
