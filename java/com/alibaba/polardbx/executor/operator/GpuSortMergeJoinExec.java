/*
 * Drop-in for SortMergeJoinExec (operator/SortMergeJoinExec.java:69-93, 109-159) backed by gsql_smj_*: joins an outer and an
 * inner input that are both ordered on the join keys and returns the rows in the stock operator's order (each outer row in
 * input order, a matched row followed by its equal-key inner rows in inner order).  The inner input is pulled to its end
 * and handed over through GpuChunks; then outer chunks are staged and probed when the stage is full, when the outer input
 * blocks and when it finishes, and each probed batch is returned in chunkLimit chunks.  The stock operator alternates
 * between its inputs; draining the inner input first is safe because the two inputs are separate exchanges or sources
 * (INTEGRATION.md).  Other conditions never reach it (GpuSupport.sortMergeJoinSupported).  Compiled where the CN is built
 * (no JDK in this repository's build image) — see INTEGRATION.md.
 */
package com.alibaba.polardbx.executor.operator;

import com.alibaba.polardbx.executor.chunk.Chunk;
import com.alibaba.polardbx.executor.chunk.GpuChunks;
import com.alibaba.polardbx.executor.operator.gpu.GpuDevices;
import com.alibaba.polardbx.executor.operator.gpu.GpuNative;
import com.alibaba.polardbx.executor.operator.gpu.GpuTypes;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.alibaba.polardbx.optimizer.core.join.EquiJoinKey;
import com.google.common.collect.ImmutableList;
import com.google.common.util.concurrent.ListenableFuture;
import org.apache.calcite.rel.core.JoinRelType;

import java.util.List;

public class GpuSortMergeJoinExec extends AbstractExecutor {
    private final Executor outerInput, innerInput;
    private final JoinRelType joinType;
    private final boolean maxOneRow;
    private final int[] outerKeys, innerKeys, keyTypes, keyDesc, antiOperands;
    private final int[] outerCodes, innerCodes;
    private final List<DataType> dataTypes;

    private long ctx, smj, innerStage, outerStage, out;
    private long left;             // rows of the probed outer batch not yet returned
    private boolean innerFinished, outerFinished;
    private ListenableFuture<?> blocked = NOT_BLOCKED;

    public GpuSortMergeJoinExec(Executor outerInput, Executor innerInput, JoinRelType joinType, boolean maxOneRow,
                                List<EquiJoinKey> joinKeys, List<Boolean> keyColumnIsAscending, int[] antiOperands,
                                List<DataType> dataTypes, ExecutionContext context) {
        super(context);
        this.outerInput = outerInput;
        this.innerInput = innerInput;
        this.joinType = joinType;
        this.maxOneRow = maxOneRow;
        this.outerKeys = joinKeys.stream().mapToInt(EquiJoinKey::getOuterIndex).toArray();
        this.innerKeys = joinKeys.stream().mapToInt(EquiJoinKey::getInnerIndex).toArray();
        this.keyTypes = joinKeys.stream().mapToInt(k -> GpuTypes.code(k.getUnifiedType())).toArray();
        this.keyDesc = keyColumnIsAscending.stream().mapToInt(asc -> asc ? 0 : 1).toArray();
        this.antiOperands = antiOperands;
        this.outerCodes = GpuTypes.codes(outerInput.getDataTypes());
        this.innerCodes = GpuTypes.codes(innerInput.getDataTypes());
        this.dataTypes = dataTypes;
    }

    @Override
    void doOpen() {
        innerInput.open();
        outerInput.open();
        ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
        smj = GpuNative.smjCreate(ctx, GpuTypes.joinType(joinType), maxOneRow, outerKeys, innerKeys, keyTypes, keyDesc,
            outerCodes, innerCodes, antiOperands);
        innerStage = GpuNative.stagingCreate(innerCodes, GpuHashAggExec.GPU_BATCH_ROWS + chunkLimit);
        outerStage = GpuNative.stagingCreate(outerCodes, GpuHashAggExec.GPU_BATCH_ROWS + chunkLimit);
        out = GpuNative.stagingCreate(GpuTypes.codes(dataTypes), chunkLimit);
    }

    private void consumeInner() {
        if (GpuNative.stagingRows(innerStage) > 0) {
            GpuNative.smjInnerConsume(smj, innerStage);
            GpuNative.stagingReset(innerStage);
        }
    }

    private void probeStaged() {
        left = GpuNative.smjProbe(smj, outerStage); // GpuMoreThanOneRowException for a single join's second match
        GpuNative.stagingReset(outerStage);
    }

    @Override
    Chunk doNextChunk() {
        while (!innerFinished) {
            Chunk chunk = innerInput.nextChunk();
            if (chunk == null) {
                if (!innerInput.produceIsFinished()) {
                    blocked = innerInput.produceIsBlocked();
                    return null; // blocked upstream: the driver will call again
                }
                consumeInner();
                GpuNative.smjInnerFinish(smj);
                innerFinished = true;
                break;
            }
            blocked = NOT_BLOCKED;
            GpuChunks.append(innerStage, chunk, innerCodes);
            if (GpuNative.stagingRows(innerStage) >= GpuHashAggExec.GPU_BATCH_ROWS) {
                consumeInner();
            }
        }
        while (left == 0 && !outerFinished) {
            Chunk chunk = outerInput.nextChunk();
            if (chunk == null) {
                if (outerInput.produceIsFinished()) {
                    outerFinished = true;
                } else if (GpuNative.stagingRows(outerStage) == 0) {
                    blocked = outerInput.produceIsBlocked();
                    return null;
                }
                if (GpuNative.stagingRows(outerStage) > 0) {
                    probeStaged();
                }
                continue;
            }
            blocked = NOT_BLOCKED;
            GpuChunks.append(outerStage, chunk, outerCodes);
            if (GpuNative.stagingRows(outerStage) >= GpuHashAggExec.GPU_BATCH_ROWS) {
                probeStaged();
            }
        }
        if (left == 0) {
            return null;
        }
        int rows = GpuNative.smjNext(smj, out, (int) Math.min(chunkLimit, left));
        left -= rows;
        // the chunk is read out of `out` before anything else writes it: the releasing call below refills `out` with 0 rows
        Chunk result = GpuChunks.toChunk(out, dataTypes, 0, rows);
        if (left == 0) {
            GpuNative.smjNext(smj, out, 0); // releases the uploaded batch now rather than at the next probe
        }
        return result;
    }

    /** Idempotent and never throws (AbstractExecutor.close). */
    @Override
    void doClose() {
        try {
            innerInput.close();
        } catch (Throwable ignored) {
        }
        try {
            outerInput.close();
        } catch (Throwable ignored) {
        }
        if (smj != 0) {
            GpuNative.smjDestroy(smj);
            GpuNative.stagingDestroy(innerStage);
            GpuNative.stagingDestroy(outerStage);
            GpuNative.stagingDestroy(out);
            GpuNative.ctxDestroy(ctx);
        }
        smj = innerStage = outerStage = out = ctx = 0;
    }

    @Override
    public List<DataType> getDataTypes() {
        return dataTypes;
    }

    @Override
    public List<Executor> getInputs() {
        return ImmutableList.of(innerInput, outerInput);
    }

    @Override
    public boolean produceIsFinished() {
        return outerFinished && left == 0;
    }

    @Override
    public ListenableFuture<?> produceIsBlocked() {
        return blocked;
    }
}
