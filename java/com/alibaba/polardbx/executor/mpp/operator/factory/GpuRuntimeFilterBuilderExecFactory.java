/*
 * GPU twin of RuntimeFilterBuilderExecFactory (mpp/operator/factory/RuntimeFilterBuilderExecFactory.java:43-115): the same
 * constructor arguments, the same filter sizing (BLOOM_FILTER_GUESS_SIZE, clamp to [BLOOM_FILTER_MIN_SIZE,
 * BLOOM_FILTER_MAX_SIZE], RuntimeFilterUtil.findMinFpp, BloomFilter.createEmpty) and the same BloomFilterProduce.create(...),
 * so the filters are sent and merged exactly as the stock ones.  It keeps the filters and MinMaxFilters it hands to the
 * BloomFilterProduce and gives them to GpuRuntimeFilterBuilderExec, which fills them from the GPU.  When the xxhash
 * parameter is off or a key / column type is not one the GPU stages (GpuSupport.runtimeFilterSupported), it creates the
 * stock RuntimeFilterBuilderExec over the same BloomFilterProduce.
 */
package com.alibaba.polardbx.executor.mpp.operator.factory;

import com.alibaba.polardbx.common.properties.ConnectionParams;
import com.alibaba.polardbx.common.utils.bloomfilter.BloomFilter;
import com.alibaba.polardbx.common.utils.hash.HashMethodInfo;
import com.alibaba.polardbx.executor.operator.Executor;
import com.alibaba.polardbx.executor.operator.GpuRuntimeFilterBuilderExec;
import com.alibaba.polardbx.executor.operator.RuntimeFilterBuilderExec;
import com.alibaba.polardbx.executor.operator.gpu.GpuSupport;
import com.alibaba.polardbx.executor.operator.util.BloomFilterProduce;
import com.alibaba.polardbx.executor.operator.util.minmaxfilter.MinMaxFilter;
import com.alibaba.polardbx.optimizer.context.ExecutionContext;
import com.alibaba.polardbx.optimizer.core.datatype.DataTypeUtil;
import com.alibaba.polardbx.optimizer.core.planner.rule.mpp.runtimefilter.RuntimeFilterUtil;
import com.alibaba.polardbx.statistics.RuntimeStatHelper;
import io.airlift.http.client.HttpClient;
import org.apache.calcite.plan.RelOptUtil;
import org.apache.calcite.rel.logical.RuntimeFilterBuilder;
import org.apache.calcite.rex.RexCall;
import org.apache.calcite.rex.RexNode;
import org.apache.calcite.rex.RexSlot;
import org.apache.calcite.sql.fun.SqlRuntimeFilterBuildFunction;

import java.net.URI;
import java.util.ArrayList;
import java.util.List;

public class GpuRuntimeFilterBuilderExecFactory extends ExecutorFactory {
    private final RuntimeFilterBuilder filterBuilder;
    private final HttpClient client;
    private final URI uri;
    private BloomFilterProduce bloomFilterProduce;
    private boolean onGpu;
    private List<BloomFilter> bloomFilters;
    private List<List<Integer>> keyHash;
    private List<List<MinMaxFilter>> minMaxFilters;

    public GpuRuntimeFilterBuilderExecFactory(RuntimeFilterBuilder filterBuilder, ExecutorFactory executorFactory,
                                              HttpClient httpClient, URI uri) {
        this.filterBuilder = filterBuilder;
        addInput(executorFactory);
        this.client = httpClient;
        this.uri = uri;
    }

    @Override
    public synchronized Executor createExecutor(ExecutionContext context, int idx) {
        Executor input = getInputs().get(0).createExecutor(context, idx);
        if (bloomFilterProduce == null) {
            boolean useXxHash = context.getParamManager().getBoolean(ConnectionParams.ENABLE_RUNTIME_FILTER_XXHASH);
            HashMethodInfo hashMethodInfo = useXxHash ? HashMethodInfo.XXHASH_METHOD : HashMethodInfo.MURMUR3_METHOD;
            keyHash = new ArrayList<>();
            bloomFilters = new ArrayList<>();
            minMaxFilters = new ArrayList<>();
            List<List<Integer>> bloomfilterId = new ArrayList<>();
            for (RexNode rexNode : RelOptUtil.conjunctions(filterBuilder.getCondition())) {
                SqlRuntimeFilterBuildFunction buildFunction = (SqlRuntimeFilterBuildFunction) ((RexCall) rexNode).getOperator();
                long ndv = Double.valueOf(buildFunction.getNdv()).longValue();
                if (context.getParamManager().getLong(ConnectionParams.BLOOM_FILTER_GUESS_SIZE) > 0) {
                    ndv = context.getParamManager().getLong(ConnectionParams.BLOOM_FILTER_GUESS_SIZE);
                }
                long size = Math.max(context.getParamManager().getLong(ConnectionParams.BLOOM_FILTER_MIN_SIZE), ndv);
                size = Math.min(context.getParamManager().getLong(ConnectionParams.BLOOM_FILTER_MAX_SIZE), size);
                double fpp = RuntimeFilterUtil.findMinFpp(ndv, size);
                List<Integer> keys = new ArrayList<>();
                List<MinMaxFilter> minMax = new ArrayList<>();
                for (RexNode operand : ((RexCall) rexNode).getOperands()) {
                    keys.add(((RexSlot) operand).getIndex());
                    minMax.add(MinMaxFilter.create(DataTypeUtil.calciteToDrdsType(operand.getType())));
                }
                bloomfilterId.add(buildFunction.getRuntimeFilterIds());
                keyHash.add(keys);
                bloomFilters.add(BloomFilter.createEmpty(hashMethodInfo, size, fpp));
                minMaxFilters.add(minMax);
            }
            bloomFilterProduce = BloomFilterProduce.create(bloomfilterId, keyHash, bloomFilters, minMaxFilters, client, uri,
                context.getTraceId());
            onGpu = GpuSupport.runtimeFilterSupported(input.getDataTypes(), keyHash, context);
            for (BloomFilter bf : bloomFilters) {
                onGpu &= bf.getNumHashFunctions() <= 64; // gsql_bloom_create: GSQL_E_UNSUPPORTED above 64
            }
        }
        bloomFilterProduce.addCounter();
        Executor exec;
        if (onGpu) {
            int[] keyColumns = new int[keyHash.size()];
            for (int i = 0; i < keyColumns.length; i++) {
                keyColumns[i] = keyHash.get(i).get(0); // one key column per filter: GpuSupport.runtimeFilterSupported
            }
            exec = new GpuRuntimeFilterBuilderExec(input, bloomFilterProduce, bloomFilters, keyColumns, minMaxFilters, context);
        } else {
            exec = new RuntimeFilterBuilderExec(input, bloomFilterProduce, context, idx);
        }
        exec.setId(filterBuilder.getRelatedId());
        if (context.getRuntimeStatistics() != null) {
            RuntimeStatHelper.registerStatForExec(filterBuilder, exec, context);
        }
        return exec;
    }
}
