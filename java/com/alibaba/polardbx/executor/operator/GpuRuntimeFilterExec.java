/*
 * Drop-in for FilterExec (operator/FilterExec.java:40-194) when its condition holds only runtime-filter calls
 * (BLOOMFILTER(key), no other predicate), backed by gsql_bloom_*.  Until the first filter arrives, chunks pass through
 * (FilterExec.java:81-84).  A filter that has arrived (BloomFilterConsume.getBloomFilter() != null) is loaded once into a
 * GPU filter of its size: gsql_bloom_merge of its getBitmap() into an empty filter, the same bits.  Then input chunks are
 * gathered into GPU_BATCH_ROWS-row batches and every loaded filter keeps the rows whose key mightContain64 accepts
 * (the filters are ANDed, as the planner's conjunction of BLOOMFILTER calls is); the surviving rows come back in
 * chunkLimit-row chunks.  The filters are xxhash_64 bitmaps (GpuSupport.runtimeFilterSupported), bit-compatible with the
 * reference's, so a filter built by a stock Java task works here unchanged.
 */
package com.alibaba.polardbx.executor.operator;

import com.alibaba.polardbx.common.utils.bloomfilter.BloomFilter;
import com.alibaba.polardbx.common.utils.hash.HashMethodInfo;
import com.alibaba.polardbx.executor.chunk.Chunk;
import com.alibaba.polardbx.executor.chunk.GpuChunks;
import com.alibaba.polardbx.executor.operator.gpu.GpuDevices;
import com.alibaba.polardbx.executor.operator.gpu.GpuExecutorException;
import com.alibaba.polardbx.executor.operator.gpu.GpuNative;
import com.alibaba.polardbx.executor.operator.gpu.GpuTypes;
import com.alibaba.polardbx.executor.operator.util.bloomfilter.BloomFilterConsume;
import com.alibaba.polardbx.executor.operator.util.bloomfilter.BloomFilterExpression;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.google.common.collect.ImmutableList;
import com.google.common.util.concurrent.ListenableFuture;

import java.util.List;

public class GpuRuntimeFilterExec extends AbstractExecutor {
    static final int GPU_BATCH_ROWS = 1 << 20;

    private final Executor input;
    private final BloomFilterExpression expression; // the FilterExecFactory's, fed by addFilter()
    private final List<BloomFilterConsume> consumes; // the consumers the expression was built from, one key column each
    private final int[] inputCodes;

    private long ctx, a, b;     // two staging batches: input, then each filter's output becomes the next one's input
    private long[] blooms;      // 0 = that filter has not arrived yet
    private long result;        // the staging batch holding the current result rows
    private int outRows, outPos;
    private boolean inputDone;

    public GpuRuntimeFilterExec(Executor input, BloomFilterExpression expression, List<BloomFilterConsume> consumes,
                                ExecutionContext context) {
        super(context);
        this.input = input;
        this.expression = expression;
        this.consumes = consumes;
        this.inputCodes = GpuTypes.codes(input.getDataTypes());
    }

    @Override
    void doOpen() {
        input.open();
        ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
        a = GpuNative.stagingCreate(inputCodes, GPU_BATCH_ROWS + chunkLimit);
        b = GpuNative.stagingCreate(inputCodes, GPU_BATCH_ROWS + chunkLimit);
        blooms = new long[consumes.size()];
    }

    /** Loads every filter that has arrived since the last batch. */
    private void loadArrivedFilters() {
        for (int i = 0; i < blooms.length; i++) {
            BloomFilter bf = consumes.get(i).getBloomFilter();
            if (blooms[i] != 0 || bf == null) {
                continue;
            }
            if (!HashMethodInfo.XXHASH_METHOD.equals(bf.getHashMethodInfo())) {
                throw new GpuExecutorException("runtime filter " + consumes.get(i).getId() + " uses " + bf.getHashMethodInfo()
                    + ": the GPU filter takes xxhash_64 only");
            }
            long[] words = bf.getBitmap();
            blooms[i] = GpuNative.bloomCreate(ctx, words.length * (long) Long.SIZE, bf.getNumHashFunctions());
            GpuNative.bloomMerge(blooms[i], words, 1);
        }
    }

    @Override
    Chunk doNextChunk() {
        if (outPos == outRows && !expression.isExistBloomFilter()) {
            return input.nextChunk();
        }
        while (outPos == outRows) { // the current result batch is used up: gather and filter the next one
            if (inputDone) {
                return null;
            }
            GpuNative.stagingReset(a);
            while (GpuNative.stagingRows(a) < GPU_BATCH_ROWS) {
                Chunk chunk = input.nextChunk();
                if (chunk == null) {
                    inputDone = input.produceIsFinished(); // a blocked producer also returns null
                    break;
                }
                GpuChunks.append(a, chunk, inputCodes);
            }
            if (GpuNative.stagingRows(a) == 0) {
                return null;
            }
            loadArrivedFilters();
            long in = a, out = b;
            outRows = GpuNative.stagingRows(a);
            for (int i = 0; i < blooms.length; i++) {
                if (blooms[i] == 0) {
                    continue; // not arrived yet: passes every row, as BloomFilterConsumeFilter.filter does
                }
                outRows = GpuNative.bloomFilter(blooms[i], in, consumes.get(i).getHashKeys().get(0), out);
                long t = in;
                in = out;
                out = t;
            }
            result = in;
            outPos = 0;
        }
        int rows = Math.min(chunkLimit, outRows - outPos);
        Chunk ret = GpuChunks.toChunk(result, input.getDataTypes(), outPos, rows);
        outPos += rows;
        return ret;
    }

    @Override
    void doClose() {
        input.close();
        if (ctx != 0) {
            for (long h : blooms) {
                GpuNative.bloomDestroy(h);
            }
            GpuNative.stagingDestroy(a);
            GpuNative.stagingDestroy(b);
            GpuNative.ctxDestroy(ctx);
            ctx = a = b = result = 0;
        }
    }

    @Override
    public List<DataType> getDataTypes() {
        return input.getDataTypes();
    }

    @Override
    public List<Executor> getInputs() {
        return ImmutableList.of(input);
    }

    @Override
    public boolean produceIsFinished() {
        return input.produceIsFinished() && outPos == outRows;
    }

    @Override
    public ListenableFuture<?> produceIsBlocked() {
        return outPos < outRows ? NOT_BLOCKED : input.produceIsBlocked();
    }
}
