/*
 * Drop-in for VectorizedFilterExec directly under VectorizedProjectExec (operator/VectorizedFilterExec.java:32-140,
 * operator/VectorizedProjectExec.java:40-143) — or for either one alone — backed by gsql_scan_*: one pass that evaluates the
 * condition, compacts the surviving rows and evaluates the output expressions (include/gsql_gpu.h: gsql_scan_spec).
 * Input chunks are gathered into GPU_BATCH_ROWS-row batches before they cross JNI; output rows come back through a staging
 * batch and are cut into chunkLimit-row chunks.  Lives in the operator package because AbstractExecutor's template methods
 * are package-private (AbstractExecutor.java:87-91).
 */
package com.alibaba.polardbx.executor.operator;

import com.alibaba.polardbx.executor.chunk.Chunk;
import com.alibaba.polardbx.executor.chunk.GpuChunks;
import com.alibaba.polardbx.executor.operator.gpu.GpuDevices;
import com.alibaba.polardbx.executor.operator.gpu.GpuExpression;
import com.alibaba.polardbx.executor.operator.gpu.GpuNative;
import com.alibaba.polardbx.executor.operator.gpu.GpuTypes;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.google.common.collect.ImmutableList;
import com.google.common.util.concurrent.ListenableFuture;

import java.util.List;

public class GpuVectorizedFilterProjectExec extends AbstractExecutor {
    static final int GPU_BATCH_ROWS = 1 << 20;

    private final Executor input;
    private final GpuExpression condition; // null: no filter (a bare Project)
    private final GpuExpression[] outputs; // one program per output column; a bare Filter passes col(i) for every column
    private final List<DataType> outputTypes;
    private final int[] inputCodes;

    private long ctx, scan, in, out;
    private int outRows, outPos;
    private boolean inputDone;

    public GpuVectorizedFilterProjectExec(Executor input, GpuExpression condition, GpuExpression[] outputs, List<DataType> outputTypes,
                                          ExecutionContext context) {
        super(context);
        this.input = input;
        this.condition = condition;
        this.outputs = outputs;
        this.outputTypes = outputTypes;
        this.inputCodes = GpuTypes.codes(input.getDataTypes());
    }

    @Override
    void doOpen() {
        input.open();
        ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
        int[][] ops = new int[outputs.length][];
        int[][] args = new int[outputs.length][];
        long[][] consts = new long[outputs.length][];
        long[][] pools = new long[outputs.length][];
        boolean create2 = condition != null && condition.needsCreate2();
        for (int i = 0; i < outputs.length; i++) {
            ops[i] = outputs[i].ops;
            args[i] = outputs[i].args;
            consts[i] = outputs[i].consts;
            pools[i] = outputs[i].pool;
            create2 |= outputs[i].needsCreate2();
        }
        if (create2) {
            scan = GpuNative.scanCreate2(ctx, inputCodes, condition == null ? null : condition.ops, condition == null ? null : condition.args,
                condition == null ? null : condition.consts, condition == null ? null : condition.pool, ops, args, consts, pools);
        } else {
            scan = GpuNative.scanCreate(ctx, inputCodes, condition == null ? null : condition.ops, condition == null ? null : condition.args,
                condition == null ? null : condition.consts, ops, args, consts);
        }
        in = GpuNative.stagingCreate(inputCodes, GPU_BATCH_ROWS + chunkLimit);
        out = GpuNative.stagingCreate(GpuTypes.codes(outputTypes), GPU_BATCH_ROWS + chunkLimit);
    }

    @Override
    Chunk doNextChunk() {
        while (outPos == outRows) { // the current result batch is used up: gather and evaluate the next one
            if (inputDone) {
                return null;
            }
            GpuNative.stagingReset(in);
            while (GpuNative.stagingRows(in) < GPU_BATCH_ROWS) {
                Chunk chunk = input.nextChunk();
                if (chunk == null) {
                    // a blocked producer also returns null: only a finished one ends the stream
                    inputDone = input.produceIsFinished();
                    break;
                }
                GpuChunks.append(in, chunk, inputCodes);
            }
            if (GpuNative.stagingRows(in) == 0) {
                if (inputDone) {
                    return null;
                }
                return null; // blocked upstream: the driver polls produceIsBlocked() and calls again
            }
            outRows = GpuNative.scanApply(scan, in, out);
            outPos = 0;
        }
        int rows = Math.min(chunkLimit, outRows - outPos);
        Chunk result = GpuChunks.toChunk(out, outputTypes, outPos, rows);
        outPos += rows;
        return result;
    }

    @Override
    void doClose() {
        input.close();
        if (scan != 0) {
            GpuNative.scanDestroy(scan);
            GpuNative.stagingDestroy(in);
            GpuNative.stagingDestroy(out);
            GpuNative.ctxDestroy(ctx);
            scan = in = out = ctx = 0;
        }
    }

    @Override
    public List<DataType> getDataTypes() {
        return outputTypes;
    }

    @Override
    public List<Executor> getInputs() {
        return ImmutableList.of(input);
    }

    @Override
    public boolean produceIsFinished() {
        return inputDone && outPos == outRows;
    }

    @Override
    public ListenableFuture<?> produceIsBlocked() {
        return outPos < outRows ? NOT_BLOCKED : input.produceIsBlocked();
    }
}
