/*
 * Drop-in for ExpandExec (operator/ExpandExec.java:39-69) + HashAggExec (operator/HashAggExec.java:74-162) backed by
 * gsql_gsagg_*: the Expand input is consumed once, never copied per grouping set.  Lives in the operator package because AbstractExecutor's template methods doOpen / doNextChunk / doClose
 * are package-private (AbstractExecutor.java:87-91).  Compiled where the CN is built (no JDK in this repository's
 * build image) — see INTEGRATION.md.
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

public class GpuExpandHashAggExec extends AbstractExecutor implements ConsumerExecutor {
    /** rows accumulated before a batch crosses JNI (GpuHashAggExec's) */
    static final int GPU_BATCH_ROWS = GpuHashAggExec.GPU_BATCH_ROWS;

    private final List<DataType> outputColumns;
    private final int[] inputCodes;       // the Expand's input: what consumeChunk receives
    private final int[] expandCodes;      // the Expand's output: what groups / spec address
    private final int[][] projSrc, projCol;
    private final long[][] projValue;
    private final int[] groups;
    private final GpuAggSpec spec; // kinds / columns / filter args derived from the plan's AggregateCalls
    private final int expectedGroups;

    private long ctx, agg, in, out;
    private boolean finished;

    /**
     * ExpandExec's arguments (its input's types, the projections, the output column types) as GpuNative.gsAggCreate takes
     * them, then HashAggExec's (groups, aggregate calls, output columns, expected groups) over the Expand's output.
     */
    public GpuExpandHashAggExec(List<DataType> inputTypes, int[][] projSrc, int[][] projCol, long[][] projValue,
                                List<DataType> expandColumns, int[] groups, GpuAggSpec spec, List<DataType> outputColumns,
                                int expectedGroups, ExecutionContext context) {
        super(context);
        this.inputCodes = GpuTypes.codes(inputTypes);
        this.expandCodes = GpuTypes.codes(expandColumns);
        this.projSrc = projSrc;
        this.projCol = projCol;
        this.projValue = projValue;
        this.groups = groups;
        this.spec = spec;
        this.outputColumns = outputColumns;
        this.expectedGroups = expectedGroups;
    }

    @Override
    public synchronized void openConsume() {
        if (agg != 0) {
            return; // LocalExchanger.openConsume opens every consumer once, but stay idempotent
        }
        ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
        agg = GpuNative.gsAggCreate(ctx, inputCodes, expandCodes, projSrc, projCol, projValue, groups, spec.kinds, spec.cols,
            spec.filterArgs, expectedGroups);
        in = GpuNative.stagingCreate(inputCodes, GPU_BATCH_ROWS + chunkLimit);
        out = GpuNative.stagingCreate(GpuTypes.codes(outputColumns), chunkLimit);
    }

    /** Several exchanger threads may feed one consumer (asyncConsume): serialised like ParallelHashJoinExec:158. */
    @Override
    public synchronized void consumeChunk(Chunk chunk) {
        GpuChunks.append(in, chunk, inputCodes); // Block arrays -> pinned staging (GetPrimitiveArrayCritical inside)
        if (GpuNative.stagingRows(in) >= GPU_BATCH_ROWS) {
            GpuNative.gsAggConsume(agg, in);
            GpuNative.stagingReset(in);
        }
    }

    @Override
    public synchronized void buildConsume() {
        if (GpuNative.stagingRows(in) > 0) {
            GpuNative.gsAggConsume(agg, in);
            GpuNative.stagingReset(in);
        }
        GpuNative.gsAggFinish(agg);
    }

    @Override
    Chunk doNextChunk() {
        int rows = GpuNative.gsAggNext(agg, out, chunkLimit);
        if (rows == 0) {
            finished = true;
            return null;
        }
        return GpuChunks.toChunk(out, outputColumns, 0, rows);
    }

    @Override
    public synchronized void closeConsume(boolean force) {
        if (agg == 0) {
            return;
        }
        GpuNative.gsAggDestroy(agg);
        GpuNative.stagingDestroy(in);
        GpuNative.stagingDestroy(out);
        GpuNative.ctxDestroy(ctx);
        agg = in = out = ctx = 0;
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
        return outputColumns;
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
