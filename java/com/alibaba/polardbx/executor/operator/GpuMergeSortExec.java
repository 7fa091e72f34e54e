/*
 * Drop-in for MergeSortExec (operator/MergeSortExec.java) backed by gsql_merge_*: the runs of its inputs, each already in
 * the order of ExecUtils.getComparator (what operator/util/MergeSortedChunks merges with ChunkWithPositionComparator),
 * come out as one sequence in that order, `offset` rows skipped and at most `limit` returned.  Same constructor
 * arguments and the same rules as the stock operator:
 *   - one input, offset 0 and limit Long.MAX_VALUE: the input's chunks pass through unchanged, no GPU work;
 *   - limit <= 0: nothing is opened and nothing returned;
 *   - otherwise every input is drained into the GPU merge (an input stops being pulled once it has delivered
 *     offset + limit rows, the most the merge keeps of it), the merge runs once all are drained, and the merged rows are
 *     handed out after skipping `offset`.
 * Rows with equal keys come out input by input (the merge is stable), a stricter order than the stock priority queue's.
 * While an input is blocked and not finished, doNextChunk returns null and produceIsBlocked reports its future.
 * Chunks are staged through one pinned buffer, flushed when it fills or the input changes.  Lives in the operator package
 * because AbstractExecutor's template methods are package-private (AbstractExecutor.java:87-91).  Compiled where the CN
 * is built (no JDK in this repository's build image) — see INTEGRATION.md.
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
import com.google.common.util.concurrent.ListenableFuture;

import java.util.List;

public class GpuMergeSortExec extends AbstractExecutor {
    private final List<Executor> inputs;
    private final long limit;
    private final long gpuLimit; // rows the merge keeps: offset + limit, or -1 (every row) when that overflows a long
    private final boolean ignoreMergeSort;
    private final int[] codes;
    private final int[] keyCols;
    private final int[] keyDesc;

    private long skipped, fetched;
    private long ctx, merge, in, out;
    private boolean[] drained;
    private long[] pulled;
    private int stagedInput = -1;
    private boolean merged, finished;
    private ListenableFuture<?> blocked = NOT_BLOCKED;

    public GpuMergeSortExec(List<Executor> inputs, List<OrderByOption> orderBys, long offset, long limit,
                            ExecutionContext context) {
        super(context);
        this.inputs = inputs;
        this.limit = limit;
        this.skipped = offset;
        this.fetched = limit;
        this.gpuLimit = gpuLimit(offset, limit);
        this.ignoreMergeSort = inputs.size() == 1 && offset == 0 && limit == Long.MAX_VALUE;
        this.codes = GpuTypes.codes(inputs.get(0).getDataTypes());
        this.keyCols = new int[orderBys.size()];
        this.keyDesc = new int[orderBys.size()];
        for (int i = 0; i < keyCols.length; i++) {
            keyCols[i] = orderBys.get(i).getIndex();
            keyDesc[i] = orderBys.get(i).isAsc() ? 0 : 1;
        }
    }

    /** offset + limit, saturating: a sum past Long.MAX_VALUE (or equal to it) means every row (-1). */
    static long gpuLimit(long offset, long limit) {
        return limit >= Long.MAX_VALUE - offset ? -1 : offset + limit;
    }

    @Override
    void doOpen() {
        if (limit <= 0) {
            return;
        }
        for (Executor input : inputs) {
            input.open();
        }
        if (!ignoreMergeSort) {
            ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
            merge = GpuNative.mergeCreate(ctx, codes, keyCols, keyDesc, inputs.size(), gpuLimit);
            in = GpuNative.stagingCreate(codes, GpuSortExec.GPU_BATCH_ROWS + chunkLimit);
            out = GpuNative.stagingCreate(codes, chunkLimit);
            drained = new boolean[inputs.size()];
            pulled = new long[inputs.size()];
        }
    }

    private void flush() {
        if (GpuNative.stagingRows(in) > 0) {
            GpuNative.mergeConsume(merge, stagedInput, in);
            GpuNative.stagingReset(in);
        }
    }

    /** Drains every input that is not blocked; true once each is finished or has delivered its quota. */
    private boolean pull() {
        blocked = NOT_BLOCKED;
        boolean all = true;
        for (int i = 0; i < inputs.size(); i++) {
            Executor input = inputs.get(i);
            while (!drained[i]) {
                Chunk chunk = input.nextChunk();
                if (chunk == null) {
                    if (input.produceIsFinished()) {
                        drained[i] = true;
                    } else if (blocked == NOT_BLOCKED) {
                        blocked = input.produceIsBlocked();
                    }
                    break;
                }
                if (stagedInput != i) {
                    flush();
                    stagedInput = i;
                }
                GpuChunks.append(in, chunk, codes);
                pulled[i] += chunk.getPositionCount();
                if (GpuNative.stagingRows(in) >= GpuSortExec.GPU_BATCH_ROWS) {
                    flush();
                }
                if (gpuLimit >= 0 && pulled[i] >= gpuLimit) {
                    drained[i] = true; // the merge keeps no more of this input
                }
            }
            all &= drained[i];
        }
        return all;
    }

    private Chunk passThrough() {
        Executor input = inputs.get(0);
        Chunk chunk = input.nextChunk();
        if (chunk == null) {
            if (input.produceIsFinished()) {
                finished = true;
            }
            blocked = input.produceIsBlocked();
        }
        return chunk;
    }

    @Override
    Chunk doNextChunk() {
        if (fetched <= 0 || finished) {
            return null;
        }
        if (ignoreMergeSort) {
            return passThrough();
        }
        if (!merged) {
            if (!pull()) {
                return null;
            }
            flush();
            GpuNative.mergeFinish(merge);
            merged = true;
        }
        while (true) {
            int rows = GpuNative.mergeNext(merge, out, chunkLimit);
            if (rows == 0) {
                finished = true;
                return null;
            }
            if (rows <= skipped) {
                skipped -= rows;
                continue;
            }
            int from = (int) skipped;
            int size = (int) Math.min(rows - skipped, fetched);
            skipped = 0;
            fetched -= size;
            return GpuChunks.toChunk(out, getDataTypes(), from, size);
        }
    }

    @Override
    void doClose() {
        if (limit <= 0) {
            return;
        }
        for (Executor input : inputs) {
            input.close();
        }
        if (merge != 0) {
            GpuNative.mergeDestroy(merge);
            GpuNative.stagingDestroy(in);
            GpuNative.stagingDestroy(out);
            GpuNative.ctxDestroy(ctx);
            merge = in = out = ctx = 0;
        }
    }

    @Override
    public List<DataType> getDataTypes() {
        return inputs.get(0).getDataTypes();
    }

    @Override
    public List<Executor> getInputs() {
        return inputs;
    }

    @Override
    public boolean produceIsFinished() {
        return fetched <= 0 || finished;
    }

    @Override
    public ListenableFuture<?> produceIsBlocked() {
        return blocked;
    }
}
