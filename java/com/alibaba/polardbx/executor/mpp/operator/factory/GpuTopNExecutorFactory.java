/*
 * GPU twin of TopNExecutorFactory (mpp/operator/factory/TopNExecutorFactory.java): same constructor arguments (minus the
 * spiller) and the same limit arithmetic — fetch and offset are read from the statement's parameters, and the operator
 * keeps topSize = skip + fetch rows (fetch = -1 without a FETCH, as the reference computes it); the Limit that
 * LocalExecutionPlanner.visitTopN puts above a TopN with an offset drops the first skip.  Selected in visitTopN when
 * GpuSupport.sortSupported(...) holds.
 */
package com.alibaba.polardbx.executor.mpp.operator.factory;

import com.alibaba.polardbx.common.jdbc.ParameterContext;
import com.alibaba.polardbx.executor.operator.Executor;
import com.alibaba.polardbx.executor.operator.GpuTopNExec;
import com.alibaba.polardbx.executor.utils.ExecUtils;
import com.alibaba.polardbx.executor.utils.OrderByOption;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.alibaba.polardbx.optimizer.core.rel.TopN;
import com.alibaba.polardbx.statistics.RuntimeStatHelper;
import org.apache.calcite.rel.RelFieldCollation;

import java.util.ArrayList;
import java.util.List;
import java.util.Map;

import static com.alibaba.polardbx.optimizer.core.planner.rule.util.CBOUtil.getRexParam;

public class GpuTopNExecutorFactory extends ExecutorFactory {
    private final TopN topN;
    private final int parallelism;
    private final List<DataType> dataTypeList;
    private final List<Executor> executors = new ArrayList<>();

    public GpuTopNExecutorFactory(TopN topN, int parallelism, List<DataType> dataTypeList) {
        this.topN = topN;
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

    /** TopNExecutorFactory's arithmetic: topSize = skip + fetch. */
    static long topSize(long skip, long fetch) {
        return skip + fetch;
    }

    private synchronized List<Executor> createAllExecutors(ExecutionContext context) {
        if (executors.isEmpty()) {
            long fetch = -1, skip = 0;
            Map<Integer, ParameterContext> params = context.getParams().getCurrentParameter();
            if (topN.fetch != null) {
                fetch = getRexParam(topN.fetch, params);
                if (topN.offset != null) {
                    skip = getRexParam(topN.offset, params);
                }
            }
            for (int j = 0; j < parallelism; j++) {
                List<RelFieldCollation> sortList = topN.getCollation().getFieldCollations();
                List<OrderByOption> orderBys = ExecUtils.convertFrom(sortList);
                GpuTopNExec exec = new GpuTopNExec(dataTypeList, orderBys, topSize(skip, fetch), context);
                exec.setId(topN.getRelatedId());
                if (context.getRuntimeStatistics() != null) {
                    RuntimeStatHelper.registerStatForExec(topN, exec, context);
                }
                executors.add(exec);
            }
        }
        return executors;
    }
}
