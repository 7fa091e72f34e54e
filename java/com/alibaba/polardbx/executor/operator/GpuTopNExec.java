/*
 * Drop-in for SpilledTopNExec (operator/SpilledTopNExec.java:60-72) backed by gsql_sort_* with a limit: the first topSize
 * rows in the order of ExecUtils.getComparator.  topSize is skip + fetch (TopNExecutorFactory); a Limit above drops
 * skip.  topSize == 0 outputs nothing; topSize < 0 is refused here exactly as the reference refuses it.  The device holds
 * O(topSize) rows: every consumed batch is cut to its best topSize rows as it arrives.  Which of several rows tied at
 * the boundary survive is unspecified, as in the reference.
 */
package com.alibaba.polardbx.executor.operator;

import com.alibaba.polardbx.executor.utils.OrderByOption;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;

import java.util.List;

public class GpuTopNExec extends GpuSortExec {
    public GpuTopNExec(List<DataType> dataTypeList, List<OrderByOption> orderBys, long topSize, ExecutionContext context) {
        super(dataTypeList, orderBys, checkTopSize(topSize), context);
    }

    private static long checkTopSize(long topSize) {
        if (topSize < 0) {
            throw new IllegalArgumentException("topN not support top size:" + topSize);
        }
        return topSize;
    }
}
