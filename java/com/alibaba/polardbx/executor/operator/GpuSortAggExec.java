/*
 * Drop-in for SortAggExec (operator/SortAggExec.java:53-112) backed by gsql_sortagg_*: one output row per run of adjacent
 * input rows whose group keys compare equal, in input order.  Pulled chunks are staged through GpuChunks and consumed when
 * the stage is full, when the input blocks and when it finishes; the groups each consume completes are returned while
 * input is still arriving.  FILTER arguments never reach it (GpuSupport.sortAggSupported).  Compiled where the CN is built
 * (no JDK in this repository's build image) — see INTEGRATION.md.
 */
package com.alibaba.polardbx.executor.operator;

import com.alibaba.polardbx.executor.chunk.Chunk;
import com.alibaba.polardbx.executor.chunk.GpuChunks;
import com.alibaba.polardbx.executor.operator.gpu.GpuAggSpec;
import com.alibaba.polardbx.executor.operator.gpu.GpuDevices;
import com.alibaba.polardbx.executor.operator.gpu.GpuNative;
import com.alibaba.polardbx.executor.operator.gpu.GpuTypes;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.google.common.collect.ImmutableList;
import com.google.common.util.concurrent.ListenableFuture;

import java.util.List;

public class GpuSortAggExec extends AbstractExecutor {
    private final Executor input;
    private final int[] groups;
    private final GpuAggSpec spec;
    private final List<DataType> outputColumnMeta;
    private final int[] inputCodes;

    private long ctx, sortAgg, in, out;
    private long ready;            // groups complete on the device and not yet returned
    private boolean inputFinished, finished;
    private ListenableFuture<?> blocked = NOT_BLOCKED;

    public GpuSortAggExec(Executor input, int[] groups, GpuAggSpec spec, List<DataType> outputColumnMeta,
                          ExecutionContext context) {
        super(context);
        this.input = input;
        this.groups = groups;
        this.spec = spec;
        this.outputColumnMeta = outputColumnMeta;
        this.inputCodes = GpuTypes.codes(input.getDataTypes());
    }

    @Override
    void doOpen() {
        input.open();
        ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
        sortAgg = GpuNative.sortAggCreate(ctx, inputCodes, groups, spec.kinds, spec.cols, spec.filterArgs);
        in = GpuNative.stagingCreate(inputCodes, GpuHashAggExec.GPU_BATCH_ROWS + chunkLimit);
        out = GpuNative.stagingCreate(GpuTypes.codes(outputColumnMeta), chunkLimit);
    }

    private void consumeStaged() {
        if (GpuNative.stagingRows(in) > 0) {
            ready = GpuNative.sortAggConsume(sortAgg, in);
            GpuNative.stagingReset(in);
        }
    }

    @Override
    Chunk doNextChunk() {
        while (ready == 0 && !inputFinished) {
            Chunk chunk = input.nextChunk();
            if (chunk == null) {
                inputFinished = input.produceIsFinished();
                blocked = input.produceIsBlocked();
                consumeStaged();
                if (inputFinished) {
                    ready = GpuNative.sortAggFinish(sortAgg);
                } else if (ready == 0) {
                    return null; // blocked upstream: the driver will call again
                }
                break;
            }
            blocked = NOT_BLOCKED;
            GpuChunks.append(in, chunk, inputCodes);
            if (GpuNative.stagingRows(in) >= GpuHashAggExec.GPU_BATCH_ROWS) {
                consumeStaged();
            }
        }
        if (ready == 0) {
            finished = inputFinished;
            return null;
        }
        int rows = GpuNative.sortAggNext(sortAgg, out, (int) Math.min(chunkLimit, ready));
        ready -= rows;
        return GpuChunks.toChunk(out, outputColumnMeta, 0, rows);
    }

    /** Idempotent and never throws (AbstractExecutor.close). */
    @Override
    void doClose() {
        try {
            input.close();
        } catch (Throwable ignored) {
        }
        if (sortAgg != 0) {
            GpuNative.sortAggDestroy(sortAgg);
            GpuNative.stagingDestroy(in);
            GpuNative.stagingDestroy(out);
            GpuNative.ctxDestroy(ctx);
        }
        sortAgg = in = out = ctx = 0;
    }

    @Override
    public List<DataType> getDataTypes() {
        return outputColumnMeta;
    }

    @Override
    public List<Executor> getInputs() {
        return ImmutableList.of(input);
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
