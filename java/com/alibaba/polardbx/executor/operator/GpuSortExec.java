/*
 * Drop-in for SortExec (operator/SortExec.java, operator/util/MemSortor.java:60-78) backed by gsql_sort_*: every consumed
 * row, handed out in the order of ExecUtils.getComparator (keys in turn, NULL the smallest value, DESC negating; the
 * collation's null direction is never read, by the reference's executor or here).  Rows with equal keys come out in
 * unspecified order, as IntArrays.quickSort leaves them.  GpuTopNExec is the same operator with a limit.  Lives in the
 * operator package because AbstractExecutor's template methods doOpen / doNextChunk / doClose are package-private
 * (AbstractExecutor.java:87-91).  Compiled where the CN is built (no JDK in this repository's build image) — see
 * INTEGRATION.md.
 */
package com.alibaba.polardbx.executor.operator;

import com.alibaba.polardbx.executor.chunk.Chunk;
import com.alibaba.polardbx.executor.chunk.GpuChunks;
import com.alibaba.polardbx.executor.operator.gpu.GpuDevices;
import com.alibaba.polardbx.executor.operator.gpu.GpuNative;
import com.alibaba.polardbx.executor.operator.gpu.GpuTypes;
import com.alibaba.polardbx.executor.utils.OrderByOption;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.google.common.collect.ImmutableList;
import com.google.common.util.concurrent.ListenableFuture;

import java.util.List;

public class GpuSortExec extends AbstractExecutor implements ConsumerExecutor {
    /** rows accumulated before a batch crosses JNI: 1000-row chunks are far too small for a kernel launch */
    static final int GPU_BATCH_ROWS = 1 << 20;

    private final List<DataType> dataTypes;
    private final int[] codes;
    private final int[] keyCols;
    private final int[] keyDesc;
    private final long limit; // -1: every row (SortExec); >= 0: topSize (SpilledTopNExec)

    private long ctx, sort, in, out;
    private boolean finished;

    public GpuSortExec(List<DataType> dataTypes, List<OrderByOption> orderBys, ExecutionContext context) {
        this(dataTypes, orderBys, -1, context);
    }

    GpuSortExec(List<DataType> dataTypes, List<OrderByOption> orderBys, long limit, ExecutionContext context) {
        super(context);
        this.dataTypes = dataTypes;
        this.codes = GpuTypes.codes(dataTypes);
        this.keyCols = new int[orderBys.size()];
        this.keyDesc = new int[orderBys.size()];
        for (int i = 0; i < keyCols.length; i++) {
            keyCols[i] = orderBys.get(i).getIndex();
            keyDesc[i] = orderBys.get(i).isAsc() ? 0 : 1;
        }
        this.limit = limit;
    }

    @Override
    public synchronized void openConsume() {
        if (sort != 0) {
            return; // LocalExchanger.openConsume opens every consumer once, but stay idempotent
        }
        ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
        sort = GpuNative.sortCreate(ctx, codes, keyCols, keyDesc, limit);
        in = GpuNative.stagingCreate(codes, GPU_BATCH_ROWS + chunkLimit);
        out = GpuNative.stagingCreate(codes, chunkLimit);
    }

    /** Several exchanger threads may feed one consumer (asyncConsume): serialised like ParallelHashJoinExec:158. */
    @Override
    public synchronized void consumeChunk(Chunk chunk) {
        GpuChunks.append(in, chunk, codes); // Block arrays -> pinned staging (GetPrimitiveArrayCritical inside)
        if (GpuNative.stagingRows(in) >= GPU_BATCH_ROWS) {
            GpuNative.sortConsume(sort, in);
            GpuNative.stagingReset(in);
        }
    }

    @Override
    public synchronized void buildConsume() {
        if (GpuNative.stagingRows(in) > 0) {
            GpuNative.sortConsume(sort, in);
            GpuNative.stagingReset(in);
        }
        GpuNative.sortFinish(sort);
    }

    @Override
    Chunk doNextChunk() {
        int rows = GpuNative.sortNext(sort, out, chunkLimit);
        if (rows == 0) {
            finished = true;
            return null;
        }
        return GpuChunks.toChunk(out, dataTypes, 0, rows);
    }

    @Override
    public synchronized void closeConsume(boolean force) {
        if (sort == 0) {
            return;
        }
        GpuNative.sortDestroy(sort);
        GpuNative.stagingDestroy(in);
        GpuNative.stagingDestroy(out);
        GpuNative.ctxDestroy(ctx);
        sort = in = out = ctx = 0;
    }

    @Override
    void doOpen() {
    }

    @Override
    void doClose() {
        closeConsume(true);
    }

    @Override
    public List<DataType> getDataTypes() {
        return dataTypes;
    }

    @Override
    public List<Executor> getInputs() {
        return ImmutableList.of();
    }

    @Override
    public boolean produceIsFinished() {
        return finished;
    }

    @Override
    public ListenableFuture<?> produceIsBlocked() {
        return NOT_BLOCKED;
    }

    @Override
    public boolean needsInput() {
        return true;
    }

    @Override
    public boolean consumeIsFinished() {
        return false;
    }

    @Override
    public ListenableFuture<?> consumeIsBlocked() {
        return ConsumerExecutor.NOT_BLOCKED;
    }
}
