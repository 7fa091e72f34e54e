/*
 * NonFrameOverWindowExec (operator/NonFrameOverWindowExec.java:60-146) backed by gsql_window_*: input chunks are staged
 * through GpuChunks and sent to the GPU GPU_BATCH_ROWS at a time (and when the input blocks or finishes); each input chunk
 * then comes back with its own blocks followed by one block per window call, every call running from the start of the
 * row's partition to the row.  It extends the stock class so that plans, statistics and instanceof checks see the operator they expect; the
 * stock aggregators are not used.  Refused shapes never reach it (GpuSupport.nonFrameWindowSupported).  Compiled where the
 * CN is built (no JDK in this repository's build image) — see INTEGRATION.md.
 */
package com.alibaba.polardbx.executor.operator;

import com.alibaba.polardbx.executor.chunk.Block;
import com.alibaba.polardbx.executor.chunk.Chunk;
import com.alibaba.polardbx.executor.chunk.GpuChunks;
import com.alibaba.polardbx.executor.operator.gpu.GpuAggSpec;
import com.alibaba.polardbx.executor.operator.gpu.GpuDevices;
import com.alibaba.polardbx.executor.operator.gpu.GpuNative;
import com.alibaba.polardbx.executor.operator.gpu.GpuTypes;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;

import com.google.common.util.concurrent.ListenableFuture;

import java.util.ArrayDeque;
import java.util.ArrayList;
import java.util.Collections;
import java.util.List;

public class GpuNonFrameOverWindowExec extends NonFrameOverWindowExec {
    private final GpuAggSpec spec;
    private final int[] partition;
    private final boolean resetEachRow;
    private final int[] inputCodes;
    private final List<DataType> callTypes;

    private long ctx, window, in, out;
    private boolean inputFinished, finished;
    private final List<Chunk> pending = new ArrayList<>();     // staged input chunks, not yet sent to the GPU
    private final ArrayDeque<Chunk> ready = new ArrayDeque<>(); // output chunks not yet returned
    private ListenableFuture<?> blocked = NOT_BLOCKED;

    /** The stock constructor's arguments, with the GpuAggSpec of the calls in place of the Aggregator list. */
    public GpuNonFrameOverWindowExec(Executor input, ExecutionContext context, GpuAggSpec spec, List<Integer> partitionIndexes,
                                     boolean resetEachRow, List<DataType> dataTypes) {
        super(input, context, Collections.emptyList(), partitionIndexes, new boolean[0], dataTypes);
        this.spec = spec;
        this.partition = partitionIndexes.stream().mapToInt(Integer::intValue).toArray();
        this.resetEachRow = resetEachRow;
        this.inputCodes = GpuTypes.codes(input.getDataTypes());
        this.callTypes = dataTypes.subList(input.getDataTypes().size(), dataTypes.size());
    }

    @Override
    void doOpen() {
        input.open();
        ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
        window = GpuNative.windowCreate(ctx, inputCodes, partition, spec.kinds, spec.cols, spec.filterArgs, resetEachRow);
        in = GpuNative.stagingCreate(inputCodes, GpuHashAggExec.GPU_BATCH_ROWS + chunkLimit);
        out = GpuNative.stagingCreate(GpuTypes.codes(callTypes), chunkLimit);
    }

    /**
     * Pulls input chunks into the staging until it holds GPU_BATCH_ROWS rows, the input blocks or it finishes, then sends
     * them to the GPU in one call; the chunks come back one by one, each with its own blocks followed by its rows of the
     * call columns, so output chunks are the input chunks, as in the stock operator.
     */
    @Override
    Chunk doNextChunk() {
        while (ready.isEmpty() && !inputFinished) {
            Chunk chunk = input.nextChunk();
            if (chunk == null) { // processStatus
                inputFinished = input.produceIsFinished();
                blocked = input.produceIsBlocked();
                flush();
                if (ready.isEmpty() && !inputFinished) {
                    return null; // blocked upstream: the driver will call again
                }
                break;
            }
            blocked = NOT_BLOCKED;
            pending.add(chunk);
            GpuChunks.append(in, chunk, inputCodes);
            if (GpuNative.stagingRows(in) >= GpuHashAggExec.GPU_BATCH_ROWS) {
                flush();
            }
        }
        Chunk next = ready.poll();
        finished = inputFinished && ready.isEmpty();
        return next;
    }

    private void flush() {
        int rows = GpuNative.stagingRows(in) > 0 ? GpuNative.windowApply(window, in, out) : 0;
        int from = 0;
        for (Chunk chunk : pending) {
            int n = chunk.getPositionCount();
            Chunk calls = GpuChunks.toChunk(out, callTypes, from, n);
            Block[] blocks = new Block[chunk.getBlockCount() + calls.getBlockCount()];
            for (int i = 0; i < chunk.getBlockCount(); i++) {
                blocks[i] = chunk.getBlock(i);
            }
            for (int i = 0; i < calls.getBlockCount(); i++) {
                blocks[chunk.getBlockCount() + i] = calls.getBlock(i);
            }
            ready.add(new Chunk(blocks));
            from += n;
        }
        assert from == rows;
        pending.clear();
        GpuNative.stagingReset(in);
    }

    /** Idempotent and never throws (AbstractExecutor.close). */
    @Override
    void doClose() {
        try {
            input.close();
        } catch (Throwable ignored) {
        }
        if (window != 0) {
            GpuNative.windowDestroy(window);
            GpuNative.stagingDestroy(in);
            GpuNative.stagingDestroy(out);
            GpuNative.ctxDestroy(ctx);
        }
        window = in = out = ctx = 0;
    }

    @Override
    public boolean produceIsFinished() {
        return finished;
    }

    @Override
    public ListenableFuture<?> produceIsBlocked() {
        return blocked;
    }
}
