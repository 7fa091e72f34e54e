/*
 * Drop-in for RuntimeFilterBuilderExec (operator/RuntimeFilterBuilderExec.java:30-98) on the build side of a runtime-filtered
 * join, backed by gsql_bloom_*: chunks pass through unchanged; the key column of every filter is gathered into a staging
 * batch and put into a GPU bloom filter (BloomFilterProduce.addChunk:92-106 does the same row by row).  The MinMaxFilter
 * updates stay on the host with the reference's own classes.  On close the GPU bitmap is ORed into the shared
 * BloomFilter's getBitmap() under that filter's lock, and only then BloomFilterProduce.close() runs, so the reference's
 * send / merge path (the last closer sends every bitmap) is reused as is.  The bitmaps are bit-compatible (xxhash_64
 * method), so parallel builders on the CPU and on the GPU may share one BloomFilterProduce.
 */
package com.alibaba.polardbx.executor.operator;

import com.alibaba.polardbx.common.utils.bloomfilter.BloomFilter;
import com.alibaba.polardbx.executor.chunk.Block;
import com.alibaba.polardbx.executor.chunk.Chunk;
import com.alibaba.polardbx.executor.chunk.GpuChunks;
import com.alibaba.polardbx.executor.operator.gpu.GpuDevices;
import com.alibaba.polardbx.executor.operator.gpu.GpuNative;
import com.alibaba.polardbx.executor.operator.gpu.GpuTypes;
import com.alibaba.polardbx.executor.operator.util.BloomFilterProduce;
import com.alibaba.polardbx.executor.operator.util.minmaxfilter.MinMaxFilter;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataType;
import com.google.common.collect.ImmutableList;
import com.google.common.util.concurrent.ListenableFuture;

import java.util.ArrayList;
import java.util.List;

public class GpuRuntimeFilterBuilderExec extends AbstractExecutor {
    static final int GPU_BATCH_ROWS = 1 << 20;

    private final Executor input;
    private BloomFilterProduce filterClient;
    private final List<BloomFilter> bloomFilters;      // the BloomFilterProduce's own filters, one per key column
    private final int[] keyColumns;                     // keyColumns[i]: the column filter i hashes
    private final List<List<MinMaxFilter>> minMaxFilters;
    private final int[] keyCodes;                       // staging types: one key column per filter

    private long ctx, staging;
    private long[] blooms;

    public GpuRuntimeFilterBuilderExec(Executor input, BloomFilterProduce filterClient, List<BloomFilter> bloomFilters,
                                       int[] keyColumns, List<List<MinMaxFilter>> minMaxFilters, ExecutionContext context) {
        super(context);
        this.input = input;
        this.filterClient = filterClient;
        this.bloomFilters = bloomFilters;
        this.keyColumns = keyColumns;
        this.minMaxFilters = minMaxFilters;
        List<DataType> types = input.getDataTypes();
        List<DataType> keyTypes = new ArrayList<>();
        for (int c : keyColumns) {
            keyTypes.add(types.get(c));
        }
        this.keyCodes = GpuTypes.codes(keyTypes);
    }

    @Override
    void doOpen() {
        input.open();
        ctx = GpuNative.ctxCreate(GpuDevices.deviceForThisDriver(context));
        staging = GpuNative.stagingCreate(keyCodes, GPU_BATCH_ROWS + chunkLimit);
        blooms = new long[bloomFilters.size()];
        for (int i = 0; i < blooms.length; i++) {
            BloomFilter bf = bloomFilters.get(i);
            blooms[i] = GpuNative.bloomCreate(ctx, bf.getBitmap().length * (long) Long.SIZE, bf.getNumHashFunctions());
        }
    }

    @Override
    Chunk doNextChunk() {
        Chunk ret = input.nextChunk();
        if (ret != null) {
            Block[] keys = new Block[keyColumns.length];
            for (int i = 0; i < keyColumns.length; i++) {
                keys[i] = ret.getBlock(keyColumns[i]);
                MinMaxFilter minMax = minMaxFilters.get(i).get(0);
                for (int pos = 0; pos < ret.getPositionCount(); pos++) {
                    minMax.put(keys[i], pos);
                }
            }
            GpuChunks.append(staging, new Chunk(ret.getPositionCount(), keys), keyCodes);
            if (GpuNative.stagingRows(staging) >= GPU_BATCH_ROWS) {
                flush();
            }
        }
        return ret;
    }

    private void flush() {
        if (GpuNative.stagingRows(staging) > 0) {
            for (int i = 0; i < blooms.length; i++) {
                GpuNative.bloomPut(blooms[i], staging, i);
            }
            GpuNative.stagingReset(staging);
        }
    }

    @Override
    void doClose() {
        try {
            if (ctx != 0) {
                flush();
                for (int i = 0; i < blooms.length; i++) {
                    BloomFilter bf = bloomFilters.get(i);
                    synchronized (bf) { // parallel builders share the filter
                        GpuNative.bloomBitmapOr(blooms[i], bf.getBitmap());
                    }
                }
            }
        } finally {
            release();
            if (filterClient != null) {
                filterClient.close(); // the last closer sends every filter (BloomFilterProduce.close:134-170)
                filterClient = null;
            }
            input.close();
        }
    }

    private void release() {
        if (ctx != 0) {
            for (long b : blooms) {
                GpuNative.bloomDestroy(b);
            }
            GpuNative.stagingDestroy(staging);
            GpuNative.ctxDestroy(ctx);
            ctx = staging = 0;
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
        return input.produceIsFinished();
    }

    @Override
    public ListenableFuture<?> produceIsBlocked() {
        return input.produceIsBlocked();
    }
}
