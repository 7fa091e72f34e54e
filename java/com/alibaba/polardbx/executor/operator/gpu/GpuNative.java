/*
 * JNI surface of libgsql_gpu.so (include/gsql_gpu.h).  jni/gsql_jni.c defines one Java_..._GpuNative_<name> per native
 * below (tests/test_jni_boundary.py checks the two lists against each other and compiles the shim against a jni.h stub;
 * the build image has no JDK, so this file itself is compiled where the CN is built).
 */
package com.alibaba.polardbx.executor.operator.gpu;

public final class GpuNative {
    static {
        System.loadLibrary("gsql_jni"); // links libgsql_gpu.so
    }

    private GpuNative() {
    }

    public static final int T_INT32 = 0, T_INT64 = 1, T_FP64 = 2, T_DEC128 = 3;

    /** gsql_ctx_create; one context per operator instance. Throws GpuExecutorException when no GPU is usable. */
    public static native long ctxCreate(int device);

    public static native void ctxDestroy(long ctx);

    /** Number of CUDA devices visible to the process (0 = the planner must keep the stock operators). */
    public static native int deviceCount();

    /**
     * A staging batch: pinned host memory owned by the native side (gsql_host_alloc), filled from Block arrays with
     * GetPrimitiveArrayCritical + memcpy.  columns[i] is int[] / long[] / double[] (IntegerBlock.intArray(),
     * LongBlock.longArray(), DoubleBlock.doubleArray()); nulls[i] is boolean[] or null (AbstractBlock.nulls()).
     * The staging remembers per column whether any appended row was NULL and hands the library `nulls = NULL`
     * otherwise (AbstractBlock.mayHaveNull() == false), so NULL-free inputs reach the packed-row fast paths.
     */
    public static native long stagingCreate(int[] types, int capacityRows);

    public static native void stagingAppend(long staging, Object[] columns, boolean[][] nulls, int arrayOffset, int rows);

    /** Same through a selection vector (Chunk.selection(), Chunk.java:57-79): row i is element selection[i]. */
    public static native void stagingAppendSelected(long staging, Object[] columns, boolean[][] nulls, int[] selection,
                                                    int rows);

    public static native int stagingRows(long staging);

    public static native void stagingReset(long staging);

    public static native void stagingDestroy(long staging);

    /** Copies rows [from, from+rows) of staged column `col` into a fresh Java array (int[] / long[] / double[]). */
    public static native Object stagingColumn(long staging, int col, int from, int rows);

    /** NULL flags of the same rows, or null when none of them is NULL. */
    public static native boolean[] stagingNulls(long staging, int col, int from, int rows);

    // ---- hash join (gsql_join_*)
    public static native long joinCreate(long ctx, int joinType, boolean maxOneRow, boolean buildOuter, int[] outerKeys,
                                         int[] innerKeys, int[] keyTypes, int[] outerTypes, int[] innerTypes,
                                         int[] antiOperands, int[] condCols, long[] condNeValues, long expectedBuildRows);

    public static native void joinBuildConsume(long join, long staging);

    public static native void joinBuildFinish(long join);

    /** Probes the staged rows; results land in `outStaging` (grown as needed). Returns the output row count. */
    public static native int joinProbe(long join, long probeStaging, long outStaging);

    public static native int joinUnmatchedBuild(long join, long outStaging);

    /** Bytes the handle holds in HBM (reported to the query MemoryPool). */
    public static native long joinDeviceBytes(long join);

    public static native void joinDestroy(long join);

    // ---- hash aggregation (gsql_agg_*)
    public static native long aggCreate(long ctx, int[] inputTypes, int[] groups, int[] aggKinds, int[][] aggCols,
                                        int[] filterArgs, long expectedGroups);

    /**
     * Same, with the Project / Filter operators that sit directly under the HashAgg fused into the kernel
     * (VectorizedProjectExec.java:40-143 / VectorizedFilterExec): derived columns {kind, a, b, c} are addressed by the
     * aggregates as input column n_input_cols + i (kind 1: a*(1-b), kind 2: a*(1-b)*(1+c)); rowFilter = {col, op, value}
     * keeps the rows with `col op value` (op: 1 <=, 2 <, 3 >=, 4 >, 5 =, 6 <>; NULL never passes), or null.
     */
    public static native long aggCreateFused(long ctx, int[] inputTypes, int[] groups, int[] aggKinds, int[][] aggCols,
                                             int[] filterArgs, long expectedGroups, int[][] derived, long[] rowFilter);

    public static native void aggConsume(long agg, long staging);

    public static native long aggFinish(long agg);

    public static native int aggNext(long agg, long outStaging, int maxRows);

    public static native void aggDestroy(long agg);

    // ---- sorted aggregation (gsql_sortagg_*): one output row per run of equal adjacent group keys, in input order
    public static native long sortAggCreate(long ctx, int[] inputTypes, int[] groups, int[] aggKinds, int[][] aggCols,
                                            int[] filterArgs);

    /** Returns the groups complete and not yet returned. */
    public static native long sortAggConsume(long sortAgg, long staging);

    /** End of input: closes the open group; returns the groups not yet returned. */
    public static native long sortAggFinish(long sortAgg);

    public static native int sortAggNext(long sortAgg, long outStaging, int maxRows);

    public static native void sortAggDestroy(long sortAgg);

    // ---- sort-merge join (gsql_smj_*): inputs ordered on the keys, rows in SortMergeJoinExec's order
    public static native long smjCreate(long ctx, int joinType, boolean maxOneRow, int[] outerKeys, int[] innerKeys,
                                        int[] keyTypes, int[] keyDesc, int[] outerTypes, int[] innerTypes, int[] antiOperands);

    public static native void smjInnerConsume(long smj, long staging);

    public static native void smjInnerFinish(long smj);

    /** Joins one outer batch; returns the exact number of rows smjNext will return for it. */
    public static native long smjProbe(long smj, long staging);

    /** Up to maxRows rows of the probed batch in order; 0 once the batch is exhausted. */
    public static native int smjNext(long smj, long outStaging, int maxRows);

    public static native void smjDestroy(long smj);

    // ---- window (gsql_window_*): NonFrameOverWindowExec, every call a running value over the row's partition
    public static native long windowCreate(long ctx, int[] inputTypes, int[] partition, int[] callKinds, int[][] callCols,
                                           int[] filterArgs, boolean resetEachRow);

    /** Writes one row per staged input row into outStaging's call columns; returns the row count. */
    public static native int windowApply(long window, long staging, long outStaging);

    public static native void windowDestroy(long window);

    // ---- vectorised filter / project (gsql_scan_*): programs are flattened {op, arg} pairs + one constant per step
    public static native long scanCreate(long ctx, int[] inputTypes, int[] filterOps, int[] filterArgs, long[] filterConsts,
                                         int[][] outOps, int[][] outArgs, long[][] outConsts);

    public static native int scanApply(long scan, long inStaging, long outStaging);

    public static native void scanDestroy(long scan);

    /**
     * PagesSerde wire format (gsql_serde_serialize): the staging batch as a stream of framed pages of at most pageRows rows
     * each — int32 positionCount | int8 marker (0 = UNCOMPRESSED) | int32 uncompressedSize | int32 sizeInBytes | raw page.
     */
    public static native byte[] serdeSerialize(long ctx, long staging, int pageRows);

    /** Decodes every framed page in pages[offset, offset + length) into outStaging (grown as needed); returns the rows. */
    public static native int serdeDeserialize(long ctx, byte[] pages, int offset, int length, long outStaging);

    // ---- local hash-partition exchange (gsql_xchg_partition)
    public static native long xchgCreate(long ctx, int[] types, int[] channels, int[] keyTypes, int nparts, int mode);

    /** Rows of `inStaging` grouped by consumer into `outStaging`; partCounts[p] = rows of consumer p. */
    public static native void xchgPartition(long xchg, long inStaging, long outStaging, long[] partCounts);

    public static native void xchgDestroy(long xchg);

    // ---- runtime bloom filter (gsql_bloom_*), bit-compatible with BloomFilter under HashMethodInfo.XXHASH_METHOD
    /** BloomFilter.createEmpty(XXHASH_METHOD, numHashFunctions, numBits). */
    public static native long bloomCreate(long ctx, long numBits, int numHashFunctions);

    /** BloomFilterProduce.addChunk: puts column keyCol of every staged row. */
    public static native void bloomPut(long bloom, long staging, int keyCol);

    /** BloomFilter.merge of nfilters getBitmap() arrays stored back to back in words. */
    public static native void bloomMerge(long bloom, long[] words, int nfilters);

    /** words |= the filter's bitmap (words = a BloomFilter's getBitmap(), under its lock). */
    public static native void bloomBitmapOr(long bloom, long[] words);

    /** FilterExec BLOOMFILTER(key): the staged rows whose key might be in the filter into outStaging; returns the rows. */
    public static native int bloomFilter(long bloom, long inStaging, int keyCol, long outStaging);

    public static native void bloomDestroy(long bloom);

    // ---- ORDER BY / TOP-N (gsql_sort_*), in the order of ExecUtils.getComparator (NULL smallest, DESC negates)
    /** SortExec (limit = -1) or SpilledTopNExec (limit = topSize = skip + fetch); keyDesc[i] = 1 for DESC. */
    public static native long sortCreate(long ctx, int[] types, int[] keyCols, int[] keyDesc, long limit);

    public static native void sortConsume(long sort, long staging);

    /** buildConsume: orders what was consumed; returns the rows sortNext will hand out. */
    public static native long sortFinish(long sort);

    /** nextChunk: up to maxRows ordered rows into outStaging; 0 = exhausted. */
    public static native int sortNext(long sort, long outStaging, int maxRows);

    public static native void sortDestroy(long sort);

    // ---- merge of sorted runs (gsql_merge_*): MergeSortExec's merge, stable across inputs
    /** nInputs runs (1..GSQL_MAX_MERGE_INPUTS), each in the keys' order; limit = -1: every row, >= 0: offset + fetch. */
    public static native long mergeCreate(long ctx, int[] types, int[] keyCols, int[] keyDesc, int nInputs, long limit);

    /** Appends the staged rows to run `input`; rows past the run's quota of `limit` are dropped. */
    public static native void mergeConsume(long merge, int input, long staging);

    /** Merges what was consumed; returns the rows mergeNext will hand out. */
    public static native long mergeFinish(long merge);

    /** Up to maxRows merged rows into outStaging; 0 = exhausted. */
    public static native int mergeNext(long merge, long outStaging, int maxRows);

    public static native void mergeDestroy(long merge);
}
