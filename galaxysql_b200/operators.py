"""Host-side mirror of the reference's operator interface for this path, on top of the C-ABI.

The reference's operators are Java (`com.alibaba.polardbx.executor.operator`); the build image has no JDK, so the
drop-in classes a maintainer would add (java/ + jni/ in this repo, see INTEGRATION.md) cannot be compiled here.
This module restates the SAME interface in Python — same class / method names, argument meaning and error
behaviour — so that the parity tests read like the reference's own (`HashJoinTest`, `HashAggExecTest`):

  Executor            EX/operator/Executor.java:27-64        open / nextChunk / close / getDataTypes / getInputs
  ProducerExecutor    EX/operator/ProducerExecutor.java:25-42 produceIsFinished / produceIsBlocked
  ConsumerExecutor    EX/operator/ConsumerExecutor.java:26-77 openConsume / consumeChunk / buildConsume / closeConsume / needsInput
  Chunk, Block        EX/chunk/Chunk.java:41-100, IntegerBlock / LongBlock / DoubleBlock
  MockExec            EXT/operator/MockExec.java:27
  GpuParallelHashJoinExec  <- EX/operator/ParallelHashJoinExec.java:64-85 (ctor), :157-166, :107-128, AbstractBufferedJoinExec.java:116-183
  GpuHashAggExec           <- EX/operator/HashAggExec.java:74-91, :133-162
  GpuPartitioningExchanger <- EX/mpp/operator/PartitioningExchanger.java:71-135

The engine hands operators CHUNK_SIZE-row chunks (default 1000, ConnectionParams.java:1088-1089); one GPU call per
16 KB would be hopeless, so consumed chunks are accumulated into large staging batches (`gpu_batch_rows`) before they
cross the ABI, and GPU output is re-sliced into <= chunkLimit-row chunks — SURVEY.md §7 "Chunk granularity".
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import api, native as N


# ------------------------------------------------------------------------------------------------- types / chunks
class DataType:
    def __init__(self, name: str, code: int, np_dtype):
        self.name, self.code, self.np = name, code, np_dtype

    def __repr__(self):
        return self.name


class DataTypes:
    IntegerType = DataType("IntegerType", N.T_INT32, np.int32)
    LongType = DataType("LongType", N.T_INT64, np.int64)
    DoubleType = DataType("DoubleType", N.T_FP64, np.float64)
    # output only: exact SUM(int|bigint) (LittleNum2DecimalSum) as a Python-int column
    DecimalType = DataType("DecimalType", N.T_DEC128, object)

    @staticmethod
    def of_code(code: int) -> DataType:
        return {N.T_INT32: DataTypes.IntegerType, N.T_INT64: DataTypes.LongType, N.T_FP64: DataTypes.DoubleType,
                N.T_DEC128: DataTypes.DecimalType}[code]


class Block:
    """values + boolean isNull (None = no nulls), EX/chunk/AbstractBlock.java:27-47."""
    dtype: DataType = None

    def __init__(self, values: np.ndarray, is_null: Optional[np.ndarray] = None):
        self.values = values
        self.is_null = is_null if (is_null is not None and is_null.any()) else None

    @classmethod
    def of(cls, *vals):
        n = len(vals)
        data = np.zeros(n, dtype=cls.dtype.np)
        nulls = np.zeros(n, dtype=bool)
        for i, v in enumerate(vals):
            if v is None:
                nulls[i] = True
            else:
                data[i] = v
        return cls(data, nulls)

    def getPositionCount(self) -> int:
        return len(self.values)

    def isNull(self, pos: int) -> bool:
        return self.is_null is not None and bool(self.is_null[pos])

    def getObject(self, pos: int):
        return None if self.isNull(pos) else self.values[pos].item() if hasattr(self.values[pos], "item") else self.values[pos]


class IntegerBlock(Block):
    dtype = DataTypes.IntegerType


class LongBlock(Block):
    dtype = DataTypes.LongType


class DoubleBlock(Block):
    dtype = DataTypes.DoubleType


class DecimalBlock(Block):
    dtype = DataTypes.DecimalType


_BLOCK_OF = {N.T_INT32: IntegerBlock, N.T_INT64: LongBlock, N.T_FP64: DoubleBlock, N.T_DEC128: DecimalBlock}


class Chunk:
    def __init__(self, *blocks: Block):
        self.blocks = list(blocks)

    def getBlock(self, i: int) -> Block:
        return self.blocks[i]

    def getBlockCount(self) -> int:
        return len(self.blocks)

    def getPositionCount(self) -> int:
        return self.blocks[0].getPositionCount() if self.blocks else 0

    def rows(self):
        return [tuple(b.getObject(r) for b in self.blocks) for r in range(self.getPositionCount())]


@dataclass
class ExecutionContext:
    chunk_size: int = 1000          # CHUNK_SIZE
    gpu_batch_rows: int = 1 << 20   # rows accumulated before a batch crosses the C-ABI
    device: int = 0
    _ctx: Optional[api.Context] = field(default=None, repr=False)

    def gpu(self) -> api.Context:
        if self._ctx is None:
            self._ctx = api.Context(self.device)
        return self._ctx


class TddlRuntimeException(RuntimeError):
    def __init__(self, error_code: str, msg: str = ""):
        super().__init__(f"{error_code}: {msg}")
        self.error_code = error_code


class ErrorCode:
    ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW = "ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW"
    ERR_EXECUTOR = "ERR_EXECUTOR"


# ------------------------------------------------------------------------------------------------- interfaces
class Executor:
    def open(self): ...
    def nextChunk(self) -> Optional[Chunk]: ...
    def close(self): ...
    def getDataTypes(self) -> List[DataType]: ...
    def getInputs(self) -> List["Executor"]:
        return []

    def produceIsFinished(self) -> bool:
        return True

    def produceIsBlocked(self):
        return NOT_BLOCKED


class ConsumerExecutor:
    def openConsume(self): ...
    def consumeChunk(self, chunk: Chunk): ...
    def buildConsume(self): ...
    def closeConsume(self, force: bool): ...

    def needsInput(self) -> bool:
        return True

    def consumeIsFinished(self) -> bool:
        return False

    def consumeIsBlocked(self):
        return NOT_BLOCKED


NOT_BLOCKED = object()  # ProducerExecutor.NOT_BLOCKED: an already-completed future


class MockExec(Executor):
    """Fake source (EXT/operator/MockExec.java:27)."""

    def __init__(self, data_types: Sequence[DataType], chunks: Sequence[Chunk]):
        self.data_types, self.chunks, self.pos = list(data_types), list(chunks), 0

    class _Builder:
        def __init__(self, types):
            self.types, self.chunks = types, []

        def withChunk(self, chunk: Chunk):
            self.chunks.append(chunk)
            return self

        def build(self):
            return MockExec(self.types, self.chunks)

    @staticmethod
    def builder(*types: DataType):
        return MockExec._Builder(list(types))

    def getChunks(self):
        return self.chunks

    def open(self):
        self.pos = 0

    def nextChunk(self):
        if self.pos < len(self.chunks):
            self.pos += 1
            return self.chunks[self.pos - 1]
        return None

    def close(self):
        pass

    def getDataTypes(self):
        return self.data_types

    def produceIsFinished(self):
        return self.pos >= len(self.chunks)


class _Staging:
    """Accumulates consumed chunks column-wise until they are handed to the GPU as one batch."""

    def __init__(self, types: Sequence[DataType]):
        self.types = list(types)
        self.parts: List[List[np.ndarray]] = [[] for _ in types]
        self.nulls: List[List[Optional[np.ndarray]]] = [[] for _ in types]
        self.rows = 0

    def add(self, chunk: Chunk):
        n = chunk.getPositionCount()
        for c, b in enumerate(chunk.blocks):
            self.parts[c].append(np.asarray(b.values, dtype=self.types[c].np))
            self.nulls[c].append(b.is_null)
        self.rows += n

    def take(self):
        cols = []
        for c, t in enumerate(self.types):
            data = np.concatenate(self.parts[c]) if self.parts[c] else np.zeros(0, t.np)
            if any(x is not None for x in self.nulls[c]):
                nl = np.concatenate([x if x is not None else np.zeros(len(p), bool) for x, p in zip(self.nulls[c], self.parts[c])])
            else:
                nl = None
            cols.append((data, nl))
        self.parts = [[] for _ in self.types]
        self.nulls = [[] for _ in self.types]
        self.rows = 0
        return cols


def _slice_chunks(cols, types: Sequence[DataType], limit: int) -> List[Chunk]:
    n = len(cols[0][0]) if cols else 0
    out = []
    for lo in range(0, n, limit):
        hi = min(n, lo + limit)
        blocks = []
        for (d, nl), t in zip(cols, types):
            if t.code == N.T_DEC128:
                vals = np.array(api.dec128_to_int(d[lo:hi]), dtype=object)
            else:
                vals = np.asarray(d[lo:hi])
            blocks.append(_BLOCK_OF[t.code](vals, None if nl is None else np.asarray(nl[lo:hi]).astype(bool)))
        out.append(Chunk(*blocks))
    return out


# ------------------------------------------------------------------------------------------------- hash join
class JoinRelType:
    INNER, LEFT, RIGHT, SEMI, ANTI = N.JOIN_INNER, N.JOIN_LEFT, N.JOIN_RIGHT, N.JOIN_SEMI, N.JOIN_ANTI


@dataclass
class EquiJoinKey:  # OPT/core/join/EquiJoinKey.java:25-48
    outerIndex: int
    innerIndex: int
    unifiedType: DataType


class GpuParallelHashJoinExec(Executor, ConsumerExecutor):
    """One object is both the build-side consumer and the probe-side producer (AbstractHashJoinExec.java:35)."""

    def __init__(self, outerInput: Executor, innerInput: Executor, joinType: int, maxOneRow: bool,
                 joinKeys: Sequence[EquiJoinKey], otherCondition=None, antiJoinOperands: Optional[Sequence[int]] = None,
                 buildOuterInput: bool = False, context: Optional[ExecutionContext] = None):
        self.outerInput, self.innerInput = outerInput, innerInput
        self.context = context or ExecutionContext()
        self.buildOuterInput = buildOuterInput
        ot = [t.code for t in outerInput.getDataTypes()]
        it = [t.code for t in innerInput.getDataTypes()]
        # otherCondition: restricted form — list of (joinRowColumn, value) meaning `col != value` (NULL-safe true)
        self.join = api.HashJoin(self.context.gpu(), joinType, ot, it, [k.outerIndex for k in joinKeys],
                                 [k.innerIndex for k in joinKeys], [k.unifiedType.code for k in joinKeys],
                                 max_one_row=maxOneRow, build_outer=buildOuterInput, anti_operands=antiJoinOperands,
                                 cond_ne=tuple(otherCondition or ()))
        self.dataTypes = [DataTypes.of_code(c) for c in self.join.out_types]
        self._build = _Staging(self.getBuildInput().getDataTypes())
        self._probe = _Staging(self.getProbeInput().getDataTypes())
        self._pending: List[Chunk] = []
        self._probe_done = False
        self._null_rows_done = False
        self._finished = False

    def getBuildInput(self) -> Executor:
        return self.outerInput if self.buildOuterInput else self.innerInput

    def getProbeInput(self) -> Executor:
        return self.innerInput if self.buildOuterInput else self.outerInput

    # ---- ConsumerExecutor (build side)
    def openConsume(self):
        pass

    def consumeChunk(self, chunk: Chunk):
        self._build.add(chunk)
        if self._build.rows >= self.context.gpu_batch_rows:
            self.join.build_consume(self._build.take())

    def buildConsume(self):
        if self._build.rows:
            self.join.build_consume(self._build.take())
        self.join.build_finish()

    def closeConsume(self, force: bool):
        pass

    # ---- Executor (probe side)
    def open(self):
        self.getProbeInput().open()

    def getDataTypes(self):
        return self.dataTypes

    def getInputs(self):
        return [self.innerInput, self.outerInput]

    def _probe_batch(self):
        cols = self._probe.take()
        try:
            out = self.join.probe(cols)
        except N.MoreThanOneRowError as e:
            raise TddlRuntimeException(ErrorCode.ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW, str(e))
        self._pending.extend(_slice_chunks(out, self.dataTypes, self.context.chunk_size))

    def nextChunk(self) -> Optional[Chunk]:
        while not self._pending and not self._finished:
            if not self._probe_done:
                ch = self.getProbeInput().nextChunk()
                if ch is not None:
                    self._probe.add(ch)
                    if self._probe.rows >= self.context.gpu_batch_rows:
                        self._probe_batch()
                    continue
                if not self.getProbeInput().produceIsFinished():
                    return None  # blocked upstream: the driver will call again
                self._probe_done = True
                if self._probe.rows:
                    self._probe_batch()
                continue
            if self.buildOuterInput and not self._null_rows_done:  # nextJoinNullRows
                self._null_rows_done = True
                self._pending.extend(_slice_chunks(self.join.unmatched_build(), self.dataTypes, self.context.chunk_size))
                continue
            self._finished = True
        return self._pending.pop(0) if self._pending else None

    def produceIsFinished(self) -> bool:
        return self._finished and not self._pending

    def close(self):  # idempotent, never throws (AbstractExecutor.java:108-120)
        try:
            self.getProbeInput().close()
            self.join.close()
        except Exception:
            pass


class GpuSortMergeJoinExec(Executor):
    """SortMergeJoinExec (EX/operator/SortMergeJoinExec.java:69-93, 109-159) over inputs ordered on the join keys
    (gsql_smj): rows come out in the stock operator's order.  The inner input is pulled to its end first, then outer chunks
    are staged up to gpu_batch_rows and probed when the stage is full, when the outer input blocks and when it finishes;
    each batch's rows are returned as chunk_size chunks.  While an input is blocked nextChunk returns None and
    produceIsBlocked is that input's.  otherCondition must be None: any other condition is refused with GsqlError
    (GSQL_E_UNSUPPORTED), as gsql_smj refuses one, so the plan keeps the stock operator."""

    def __init__(self, outerInput: Executor, innerInput: Executor, joinType: int, maxOneRow: bool,
                 joinKeys: Sequence[EquiJoinKey], keyColumnIsAscending: Sequence[bool], otherCondition=None,
                 antiJoinOperands: Optional[Sequence[int]] = None, context: Optional[ExecutionContext] = None):
        if otherCondition is not None:
            raise N.GsqlError(N.E_UNSUPPORTED, "sort-merge join with another condition: the stock operator keeps it")
        self.outerInput, self.innerInput = outerInput, innerInput
        self.context = context or ExecutionContext()
        self.join = api.SortMergeJoin(self.context.gpu(), joinType, [t.code for t in outerInput.getDataTypes()],
                                      [t.code for t in innerInput.getDataTypes()], [k.outerIndex for k in joinKeys],
                                      [k.innerIndex for k in joinKeys], [k.unifiedType.code for k in joinKeys],
                                      desc=[not a for a in keyColumnIsAscending], max_one_row=maxOneRow,
                                      anti_operands=antiJoinOperands)
        self.dataTypes = [DataTypes.of_code(c) for c in self.join.out_types]
        self._inner = _Staging(innerInput.getDataTypes())
        self._outer = _Staging(outerInput.getDataTypes())
        self._inner_done = self._outer_done = False
        self._left = 0  # rows of the probed outer batch not yet returned
        self._blocked = NOT_BLOCKED
        self._closed = False

    def getDataTypes(self):
        return self.dataTypes

    def getInputs(self):
        return [self.innerInput, self.outerInput]

    def open(self):
        self.innerInput.open()
        self.outerInput.open()

    def _probe(self):
        try:
            self._left = self.join.probe(self._outer.take())
        except N.MoreThanOneRowError as e:
            raise TddlRuntimeException(ErrorCode.ERR_SCALAR_SUBQUERY_RETURN_MORE_THAN_ONE_ROW, str(e))

    def _pull_inner(self) -> bool:
        while not self._inner_done:
            ch = self.innerInput.nextChunk()
            if ch is None:
                if not self.innerInput.produceIsFinished():
                    self._blocked = self.innerInput.produceIsBlocked()
                    return False
                if self._inner.rows:
                    self.join.inner_consume(self._inner.take())
                self.join.inner_finish()
                self._inner_done = True
                break
            self._blocked = NOT_BLOCKED
            self._inner.add(ch)
            if self._inner.rows >= self.context.gpu_batch_rows:
                self.join.inner_consume(self._inner.take())
        return True

    def nextChunk(self) -> Optional[Chunk]:
        if not self._pull_inner():
            return None  # blocked upstream: the driver will call again
        while self._left == 0 and not self._outer_done:
            ch = self.outerInput.nextChunk()
            if ch is None:
                if self.outerInput.produceIsFinished():
                    self._outer_done = True
                elif not self._outer.rows:
                    self._blocked = self.outerInput.produceIsBlocked()
                    return None
                if self._outer.rows:
                    self._probe()
                continue
            self._blocked = NOT_BLOCKED
            self._outer.add(ch)
            if self._outer.rows >= self.context.gpu_batch_rows:
                self._probe()
        if self._left == 0:
            return None
        cols = self.join.next(min(self._left, self.context.chunk_size))
        self._left -= len(cols[0][0])
        return _slice_chunks(cols, self.dataTypes, self.context.chunk_size)[0]

    def produceIsFinished(self) -> bool:
        return self._outer_done and self._left == 0

    def produceIsBlocked(self):
        return self._blocked

    def close(self):  # idempotent, never throws (AbstractExecutor.java:108-120)
        if self._closed:
            return
        self._closed = True
        for x in (self.innerInput, self.outerInput, self.join):
            try:
                x.close()
            except Exception:
                pass


# ------------------------------------------------------------------------------------------------- hash agg
@dataclass
class Aggregator:
    kind: int
    targetIndexes: Sequence[int] = ()
    filterArg: int = -1


def CountRow(filterArg: int = -1):
    return Aggregator(N.AGG_COUNT_STAR, (), filterArg)


def Count(targetIndexes: Sequence[int], isDistinct: bool = False, filterArg: int = -1):
    assert not isDistinct, "DISTINCT aggregates stay on the stock operator"
    return Aggregator(N.AGG_COUNT, tuple(targetIndexes), filterArg)


def Sum(index: int, isDistinct: bool = False, outputType=None, filterArg: int = -1):
    assert not isDistinct
    return Aggregator(N.AGG_SUM, (index,), filterArg)


def Avg(index: int, isDistinct: bool = False, outputType=None, filterArg: int = -1):
    assert not isDistinct
    return Aggregator(N.AGG_AVG, (index,), filterArg)


def Min(index: int, filterArg: int = -1):
    return Aggregator(N.AGG_MIN, (index,), filterArg)


def Max(index: int, filterArg: int = -1):
    return Aggregator(N.AGG_MAX, (index,), filterArg)


def Sum0(index: int, filterArg: int = -1):
    return Aggregator(N.AGG_SUM0, (index,), filterArg)


def InternalFirstValue(index: int, outType=None, filterArg: int = -1):
    """__FIRST_VALUE (InternalFirstValue): the output type is the input's.  A filterArg >= 0 is refused when the
    executor is built (GSQL_E_UNSUPPORTED), as the stock aggregator cannot run one either."""
    return Aggregator(N.AGG_FIRST_VALUE, (index,), filterArg)



def RowNumber(filterArg: int = -1):
    """ROW_NUMBER (EX/calc/aggfunctions/RowNumber.java): window operator only."""
    return Aggregator(N.AGG_ROW_NUMBER, (), filterArg)


def Rank(index: Sequence[int] = (), filterArg: int = -1):
    """RANK over the peer (ORDER BY) columns `index` (EX/calc/aggfunctions/Rank.java): window operator only."""
    return Aggregator(N.AGG_RANK, tuple(index) if len(index) and index[0] >= 0 else (), filterArg)


def DenseRank(index: Sequence[int] = (), filterArg: int = -1):
    """DENSE_RANK (EX/calc/aggfunctions/DenseRank.java): window operator only."""
    return Aggregator(N.AGG_DENSE_RANK, tuple(index) if len(index) and index[0] >= 0 else (), filterArg)

class GpuHashAggExec(Executor, ConsumerExecutor):
    def __init__(self, inputDataTypes: Sequence[DataType], groups: Sequence[int], aggregators: Sequence[Aggregator],
                 outputColumns: Optional[Sequence[DataType]] = None, expectedGroups: int = 1024,
                 context: Optional[ExecutionContext] = None):
        self.context = context or ExecutionContext()
        self.inputDataTypes = list(inputDataTypes)
        self.agg = api.HashAgg(self.context.gpu(), [t.code for t in inputDataTypes], list(groups),
                               [(a.kind, list(a.targetIndexes)) for a in aggregators], expectedGroups,
                               filter_args=[a.filterArg for a in aggregators])
        self.dataTypes = [DataTypes.of_code(c) for c in self.agg.out_types]
        self._stage = _Staging(self.inputDataTypes)
        self._result: Optional[List[Chunk]] = None
        self._finished = False

    def openConsume(self):
        pass

    def consumeChunk(self, chunk: Chunk):
        self._stage.add(chunk)
        if self._stage.rows >= self.context.gpu_batch_rows:
            self.agg.consume(self._stage.take())

    def buildConsume(self):
        if self._stage.rows:
            self.agg.consume(self._stage.take())
        self._result = _slice_chunks(self.agg.result(), self.dataTypes, self.context.chunk_size)

    def closeConsume(self, force: bool):
        pass

    def open(self):
        pass

    def getDataTypes(self):
        return self.dataTypes

    def nextChunk(self):
        if self._result:
            return self._result.pop(0)
        self._finished = True
        return None

    def produceIsFinished(self):
        return self._finished

    def close(self):
        try:
            self.agg.close()
        except Exception:
            pass


class GpuSortAggExec(Executor):
    """SortAggExec (EX/operator/SortAggExec.java:53-112): aggregates runs of adjacent rows with equal group keys of an input
    ordered on them (gsql_sortagg).  Pulled chunks are staged up to gpu_batch_rows and consumed when the stage is full, when
    the input blocks and when it finishes; the groups each consume completes are returned as chunk_size chunks while input
    is still arriving.  While the input is blocked nextChunk returns None and produceIsBlocked is the input's."""

    def __init__(self, input: Executor, groups: Sequence[int], aggregators: Sequence[Aggregator],
                 outputColumnMeta: Optional[Sequence[DataType]] = None, context: Optional[ExecutionContext] = None):
        self.input = input
        self.context = context or ExecutionContext()
        self.agg = api.SortAgg(self.context.gpu(), [t.code for t in input.getDataTypes()], list(groups),
                               [(a.kind, list(a.targetIndexes)) for a in aggregators],
                               filter_args=[a.filterArg for a in aggregators])
        self.gpuTypes = [DataTypes.of_code(c) for c in self.agg.out_types]
        self.outputColumnMeta = list(outputColumnMeta) if outputColumnMeta is not None else self.gpuTypes
        self._stage = _Staging(input.getDataTypes())
        self._pending: List[Chunk] = []
        self._input_done = False
        self._blocked = NOT_BLOCKED
        self._closed = False

    def getDataTypes(self):
        return self.outputColumnMeta

    def getInputs(self):
        return [self.input]

    def open(self):
        self.input.open()

    def _consume(self, final: bool):
        ready = self.agg.consume(self._stage.take()) if self._stage.rows else 0
        if final:
            ready = self.agg.finish()
        if ready:
            self._pending.extend(_slice_chunks(self.agg.next(ready), self.gpuTypes, self.context.chunk_size))

    def nextChunk(self) -> Optional[Chunk]:
        while not self._pending and not self._input_done:
            ch = self.input.nextChunk()
            if ch is None:
                self._blocked = self.input.produceIsBlocked()
                self._input_done = self.input.produceIsFinished()
                self._consume(final=self._input_done)
                if not self._input_done:
                    break  # blocked upstream: the driver will call again
                continue
            self._blocked = NOT_BLOCKED
            self._stage.add(ch)
            if self._stage.rows >= self.context.gpu_batch_rows:
                self._consume(final=False)
        return self._pending.pop(0) if self._pending else None

    def produceIsFinished(self) -> bool:
        return self._input_done and not self._pending

    def produceIsBlocked(self):
        return self._blocked

    def close(self):  # idempotent, never throws (AbstractExecutor.java:108-120)
        if self._closed:
            return
        self._closed = True
        try:
            self.input.close()
        except Exception:
            pass
        try:
            self.agg.close()
        except Exception:
            pass



class GpuNonFrameOverWindowExec(Executor):
    """NonFrameOverWindowExec (EX/operator/NonFrameOverWindowExec.java:60-146): one output chunk per input chunk, the
    input's blocks followed by one block per window call (gsql_window), each call running from the start of the row's
    partition to the row.  Input chunks are staged up to gpu_batch_rows and sent to the GPU in one call when the stage is
    full, when the input blocks and when it finishes.  resetAccumulators holds the one flag of the group's frame for every
    call (the factory sets all of them alike); calls that differ are refused with GSQL_E_UNSUPPORTED, as are FILTER
    arguments."""

    def __init__(self, input: Executor, context: Optional[ExecutionContext], aggregators: Sequence[Aggregator],
                 partitionIndexes: Sequence[int], resetAccumulators: Sequence[bool], dataTypes: Sequence[DataType]):
        self.input = input
        self.context = context or ExecutionContext()
        reset = [bool(r) for r in resetAccumulators]
        if len(set(reset)) > 1:
            raise N.GsqlError(N.E_UNSUPPORTED, "window: calls with different frames")
        self.win = api.Window(self.context.gpu(), [t.code for t in input.getDataTypes()], list(partitionIndexes),
                              [(a.kind, list(a.targetIndexes)) for a in aggregators], reset_each_row=bool(reset and reset[0]),
                              filter_args=[a.filterArg for a in aggregators])
        self.callTypes = [DataTypes.of_code(c) for c in self.win.out_types]
        self.dataTypes = list(dataTypes)
        self._stage = _Staging(input.getDataTypes())
        self._pendingIn: List[Chunk] = []  # staged input chunks, not yet sent to the GPU
        self._ready: List[Chunk] = []      # output chunks not yet returned
        self._inputDone = False
        self._finished = False
        self._blocked = NOT_BLOCKED
        self._closed = False

    def getDataTypes(self):
        return self.dataTypes

    def getInputs(self):
        return [self.input]

    def open(self):
        self.input.open()

    def _flush(self):
        res = self.win.apply(self._stage.take()) if self._stage.rows else None
        lo = 0
        for ch in self._pendingIn:
            n = ch.getPositionCount()
            if n == 0:
                calls = [_BLOCK_OF[t.code](np.zeros(0, t.np)) for t in self.callTypes]
            else:
                calls = _slice_chunks([(d[lo:lo + n], nl[lo:lo + n]) for d, nl in res], self.callTypes, n)[0].blocks
            self._ready.append(Chunk(*ch.blocks, *calls))
            lo += n
        self._pendingIn = []

    def nextChunk(self) -> Optional[Chunk]:
        while not self._ready and not self._inputDone:
            ch = self.input.nextChunk()
            if ch is None:
                self._inputDone = self.input.produceIsFinished()
                self._blocked = self.input.produceIsBlocked()
                self._flush()
                if not self._inputDone and not self._ready:
                    return None  # blocked upstream: the driver will call again
                break
            self._blocked = NOT_BLOCKED
            self._pendingIn.append(ch)
            self._stage.add(ch)
            if self._stage.rows >= self.context.gpu_batch_rows:
                self._flush()
        out = self._ready.pop(0) if self._ready else None
        self._finished = self._inputDone and not self._ready
        return out

    def produceIsFinished(self) -> bool:
        return self._finished

    def produceIsBlocked(self):
        return self._blocked

    def close(self):  # idempotent, never throws (AbstractExecutor.java:108-120)
        if self._closed:
            return
        self._closed = True
        try:
            self.input.close()
        except Exception:
            pass
        try:
            self.win.close()
        except Exception:
            pass

# ------------------------------------------------------------------------------------------------- sort / top-n
class Direction:  # org.apache.calcite.rel.RelFieldCollation.Direction
    ASCENDING, DESCENDING = "ASCENDING", "DESCENDING"


class NullDirection:  # RelFieldCollation.NullDirection: carried, never read by the executor's comparator
    FIRST, LAST, UNSPECIFIED = "FIRST", "LAST", "UNSPECIFIED"


@dataclass
class OrderByOption:  # EX/utils/OrderByOption.java
    index: int
    direction: str = Direction.ASCENDING
    nullDirection: str = NullDirection.UNSPECIFIED

    def isAsc(self) -> bool:
        return self.direction == Direction.ASCENDING


class _GpuOrderExec(Executor, ConsumerExecutor):
    """Shared body of GpuSortExec / GpuTopNExec: consumed chunks are staged into large batches, ordered on the GPU by
    buildConsume, and handed out in <= chunk_size-row chunks."""

    def __init__(self, dataTypes: Sequence[DataType], orderBys: Sequence[OrderByOption], limit: Optional[int],
                 context: Optional[ExecutionContext]):
        self.context = context or ExecutionContext()
        self.dataTypes = list(dataTypes)
        self.sort = api.Sort(self.context.gpu(), [t.code for t in self.dataTypes], [o.index for o in orderBys],
                             [not o.isAsc() for o in orderBys], limit)
        self._stage = _Staging(self.dataTypes)
        self._result: Optional[List[Chunk]] = None
        self._finished = False

    def openConsume(self):
        pass

    def consumeChunk(self, chunk: Chunk):
        self._stage.add(chunk)
        if self._stage.rows >= self.context.gpu_batch_rows:
            self.sort.consume(self._stage.take())

    def buildConsume(self):
        if self._stage.rows:
            self.sort.consume(self._stage.take())
        self._result = _slice_chunks(self.sort.result(), self.dataTypes, self.context.chunk_size)

    def closeConsume(self, force: bool):
        pass

    def open(self):
        pass

    def getDataTypes(self):
        return self.dataTypes

    def nextChunk(self):
        if self._result:
            return self._result.pop(0)
        self._finished = True
        return None

    def produceIsFinished(self):
        return self._finished

    def close(self):
        try:
            self.sort.close()
        except Exception:
            pass


class GpuSortExec(_GpuOrderExec):
    """SortExec (EX/operator/SortExec.java, MemSortor.java:60-78): every row, in the executor comparator's order."""

    def __init__(self, dataTypes: Sequence[DataType], orderBys: Sequence[OrderByOption], context: Optional[ExecutionContext] = None,
                 spillerFactory=None):
        super().__init__(dataTypes, orderBys, None, context)


class GpuTopNExec(_GpuOrderExec):
    """SpilledTopNExec (EX/operator/SpilledTopNExec.java:60-72): the first topSize rows (TopNExecutorFactory passes
    skip + fetch); topSize == 0 passes nothing, topSize < 0 is an IllegalArgumentException."""

    def __init__(self, dataTypes: Sequence[DataType], orderBys: Sequence[OrderByOption], topSize: int,
                 context: Optional[ExecutionContext] = None):
        if topSize < 0:
            raise ValueError(f"topN not support top size:{topSize}")
        super().__init__(dataTypes, orderBys, topSize, context)


LONG_MAX = (1 << 63) - 1


def merge_gpu_limit(offset: int, limit: int) -> Optional[int]:
    """The rows a merge must produce for OFFSET offset FETCH limit: offset + limit, None (every row) when the sum
    overflows a long or limit is Long.MAX_VALUE with no offset."""
    total = offset + limit
    return None if total >= LONG_MAX else total


class GpuMergeSortExec(Executor):
    """MergeSortExec (EX/operator/MergeSortExec.java): merges its inputs' runs, each already in the executor comparator's
    order, skips `offset` rows and returns at most `limit`.  Inputs are pulled until each is finished or has delivered
    offset + limit rows; while one is blocked nextChunk returns None and resumes on the next call.  The merge runs on the
    GPU once every input is drained (gsql_merge, stable).  One input with offset 0 and limit Long.MAX_VALUE passes its
    chunks through untouched; limit <= 0 opens nothing and returns nothing."""

    def __init__(self, inputs: Sequence[Executor], orderBys: Sequence[OrderByOption], offset: int, limit: int,
                 context: Optional[ExecutionContext] = None):
        self.context = context or ExecutionContext()
        self.inputs, self.orderBys = list(inputs), list(orderBys)
        self.limit, self.skipped, self.fetched = limit, offset, limit
        self.ignoreMergeSort = len(self.inputs) == 1 and offset == 0 and limit == LONG_MAX
        self.gpu_limit = merge_gpu_limit(offset, limit) if limit > 0 else 0
        self.merge: Optional[api.Merge] = None
        self._done: List[bool] = []
        self._taken: List[int] = []
        self._stage: Optional[_Staging] = None
        self._stage_input = -1
        self._result: Optional[List[Chunk]] = None
        self._finished = False
        self._blocked = NOT_BLOCKED

    def getDataTypes(self):
        return self.inputs[0].getDataTypes()

    def getInputs(self):
        return self.inputs

    def open(self):
        if self.limit <= 0:
            return
        for x in self.inputs:
            x.open()
        if not self.ignoreMergeSort:
            types = self.getDataTypes()
            self.merge = api.Merge(self.context.gpu(), [t.code for t in types], [o.index for o in self.orderBys],
                                   [not o.isAsc() for o in self.orderBys], len(self.inputs), self.gpu_limit)
            self._done = [False] * len(self.inputs)
            self._taken = [0] * len(self.inputs)
            self._stage = _Staging(types)

    def _flush(self):
        if self._stage.rows:
            self.merge.consume(self._stage_input, self._stage.take())

    def _pull(self) -> bool:
        """Drains every input that is not blocked; True once all are finished or have delivered their quota."""
        self._blocked = NOT_BLOCKED
        for i, x in enumerate(self.inputs):
            while not self._done[i]:
                ch = x.nextChunk()
                if ch is None:
                    if x.produceIsFinished():
                        self._done[i] = True
                    elif self._blocked is NOT_BLOCKED:
                        self._blocked = x.produceIsBlocked()
                    break
                if self._stage_input != i:
                    self._flush()
                    self._stage_input = i
                self._stage.add(ch)
                self._taken[i] += ch.getPositionCount()
                if self._stage.rows >= self.context.gpu_batch_rows:
                    self._flush()
                if self.gpu_limit is not None and self._taken[i] >= self.gpu_limit:
                    self._done[i] = True  # the merge keeps no more of this input
        return all(self._done)

    def _merged(self) -> List[Chunk]:
        self._flush()
        cols = self.merge.result()
        lo = min(self.skipped, len(cols[0][0]))
        hi = min(len(cols[0][0]), lo + self.fetched)
        self.skipped, self.fetched = 0, self.fetched - (hi - lo)
        cols = [(d[lo:hi], None if nl is None else nl[lo:hi]) for d, nl in cols]
        return _slice_chunks(cols, self.getDataTypes(), self.context.chunk_size)

    def _passthrough(self) -> Optional[Chunk]:
        ch = self.inputs[0].nextChunk()
        if ch is None:
            if self.inputs[0].produceIsFinished():
                self._finished = True
            self._blocked = self.inputs[0].produceIsBlocked()
            return None
        self.fetched -= ch.getPositionCount()
        return ch

    def nextChunk(self) -> Optional[Chunk]:
        if self.limit <= 0 or self._finished:
            return None
        if self.ignoreMergeSort:
            return self._passthrough()
        if self._result is None:
            if not self._pull():
                return None
            self._result = self._merged()
        if self._result:
            return self._result.pop(0)
        self._finished = True
        return None

    def produceIsFinished(self) -> bool:
        return self.limit <= 0 or self._finished

    def produceIsBlocked(self):
        return self._blocked

    def close(self):
        if self.limit <= 0:
            return
        for x in self.inputs:
            x.close()
        if self.merge is not None:
            try:
                self.merge.close()
            except Exception:
                pass
            self.merge = None


# ------------------------------------------------------------------------------------------------- local exchange
class GpuPartitioningExchanger(ConsumerExecutor):
    """LocalExchange(PARTITION): routes every row to executors[partition(hash(keys))] (PartitioningExchanger.java:71-135)."""

    def __init__(self, executors: Sequence[ConsumerExecutor], types: Sequence[DataType], partitionChannels: Sequence[int],
                 context: Optional[ExecutionContext] = None):
        self.executors, self.types = list(executors), list(types)
        self.context = context or ExecutionContext()
        self.x = api.Exchange(self.context.gpu(), [t.code for t in types], list(partitionChannels), len(executors))
        self._stage = _Staging(self.types)

    def openConsume(self):
        for e in self.executors:
            e.openConsume()

    def _flush(self):
        cols, counts = self.x.partition(self._stage.take())
        off = 0
        for p, cnt in enumerate(counts.tolist()):
            if cnt:
                part = [(d[off:off + cnt], None if nl is None else nl[off:off + cnt]) for d, nl in cols]
                for ch in _slice_chunks(part, self.types, self.context.chunk_size):
                    self.executors[p].consumeChunk(ch)
            off += cnt

    def consumeChunk(self, chunk: Chunk):
        self._stage.add(chunk)
        if self._stage.rows >= self.context.gpu_batch_rows:
            self._flush()

    def buildConsume(self):
        if self._stage.rows:
            self._flush()
        for e in self.executors:  # LocalExchanger.buildConsume:97-121 fans out exactly once
            e.buildConsume()

    def closeConsume(self, force: bool):
        for e in self.executors:
            e.closeConsume(force)
        self.x.close()


# ------------------------------------------------------------------------------------------------- test driver
class SingleExecTest:
    """Serial consume -> buildConsume -> serial produce (EXT/operator/ExecTestDriver.java:97-135)."""

    def __init__(self, exec_: Executor, consumer_input: Optional[Executor] = None, chunks: Optional[Sequence[Chunk]] = None):
        self.exec_, self.consumer_input, self.chunks = exec_, consumer_input, chunks
        self._result: List[Chunk] = []

    def exec(self):
        consumer = self.exec_ if isinstance(self.exec_, ConsumerExecutor) else None
        if consumer is not None:
            consumer.openConsume()
            if self.consumer_input is not None:
                self.consumer_input.open()
                while True:
                    ch = self.consumer_input.nextChunk()
                    if ch is None:
                        break
                    consumer.consumeChunk(ch)
            for ch in self.chunks or []:
                consumer.consumeChunk(ch)
            consumer.buildConsume()
        self.exec_.open()
        while True:
            ch = self.exec_.nextChunk()
            if ch is None:
                if self.exec_.produceIsFinished():
                    break
                continue
            self._result.append(ch)
        self.exec_.close()
        return self

    def result(self) -> List[Chunk]:
        return self._result
