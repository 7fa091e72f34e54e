"""Seeded hash-join cases shared by test_hash_join_ref_cpu.py (reference vs oracle) and test_join_semantics_gpu.py
(GPU vs reference): every join mode, key type and widening, key edge value and build shape the generic join path
has to get right.

A case is a dict: ``id``, ``spec`` (oracle.JoinSpec), ``outer`` / ``inner`` columns, ``build_parts`` /
``probe_parts`` (how many batches the GPU run splits each side into; a probe split always includes an empty batch),
and ``oracle``: False where the oracle's answer depends on its hash layout (a -0.0 and a +0.0 key in one join) or
its RIGHT single-join row builder writes a different column order than its own schema.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np

from oracle import oracle as orc
from tests import kat_util as ku

I32, I64, F64 = orc.T_INT32, orc.T_INT64, orc.T_FP64
INNER, LEFT, RIGHT, SEMI, ANTI = orc.JOIN_INNER, orc.JOIN_LEFT, orc.JOIN_RIGHT, orc.JOIN_SEMI, orc.JOIN_ANTI
JT_NAME = {INNER: "inner", LEFT: "left", RIGHT: "right", SEMI: "semi", ANTI: "anti"}
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1


def f64_array(bits: List[int]) -> np.ndarray:
    """Doubles from their bit patterns (NaN payloads kept: no arithmetic touches them)."""
    return np.array([b & (2**64 - 1) for b in bits], dtype=np.uint64).view(np.float64)


# special doubles by bit pattern: quiet / signalling / negative NaNs with payloads, ±Inf, subnormals, extremes
NANS = [0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000000, 0x7FFFFFFFFFFFFFFF, 0xFFF00000DEADBEEF]
FINITE_SPECIALS = [0x7FF0000000000000, 0xFFF0000000000000,      # +Inf, -Inf
                   0x0000000000000001, 0x8000000000000001,      # ±smallest subnormal
                   0x000FFFFFFFFFFFFF, 0x0010000000000000,      # largest subnormal, smallest normal
                   0x7FEFFFFFFFFFFFFF, 0x3FF0000000000000, 0xBFF0000000000000, 0x4340000000000000]  # max, ±1, 2^53
POS_ZERO, NEG_ZERO = 0x0000000000000000, 0x8000000000000000


def rcol(n: int, seed: int, dtype, mod: int, null_frac: float = 0.0, offset: int = 0) -> "ku.Col":
    v = (ku.rand_u64(n, seed) % np.uint64(mod)).astype(np.int64) + offset
    return ku.with_nulls(v.astype(dtype), null_frac, seed + 7777)


def pick(values: np.ndarray, n: int, seed: int, null_frac: float = 0.0) -> "ku.Col":
    """n draws (with repetition) from `values`, bit-preserving."""
    idx = (ku.rand_u64(n, seed) % np.uint64(len(values))).astype(np.int64)
    return ku.with_nulls(values[idx], null_frac, seed + 7777)


def spec(jt, okeys, ikeys, ktypes, **kw) -> "orc.JoinSpec":
    return orc.JoinSpec(jt, list(okeys), list(ikeys), list(ktypes), **kw)


def case(id_, sp, outer, inner, build_parts=1, probe_parts=1, oracle=True) -> dict:
    if sp.max_one_row and sp.join_type == RIGHT:
        oracle = False
    return dict(id=id_, spec=sp, outer=outer, inner=inner, build_parts=build_parts, probe_parts=probe_parts,
                oracle=oracle)


# ---------------------------------------------------------------------------------------------- tables
def mixed_tables(n_out: int, n_in: int, key_mod: int, null_frac: float, seed: int):
    """outer: (k INT64, a INT32, p INT64, d DOUBLE); inner: (k INT64, b INT32, q INT32, e DOUBLE).  Keys repeat on
    both sides; every column but the doubles carries NULLs; the doubles are special values (NaNs, ±0.0, ±Inf, ...)."""
    specials = f64_array(FINITE_SPECIALS + NANS + [NEG_ZERO, POS_ZERO])
    outer = [rcol(n_out, seed, np.int64, key_mod, null_frac, -key_mod // 3),
             rcol(n_out, seed + 1, np.int32, 7, null_frac),
             rcol(n_out, seed + 2, np.int64, 1 << 40, null_frac, -(1 << 39)),
             pick(specials, n_out, seed + 3)]
    inner = [rcol(n_in, seed + 10, np.int64, key_mod, null_frac, -key_mod // 3),
             rcol(n_in, seed + 11, np.int32, 5, null_frac),
             rcol(n_in, seed + 12, np.int32, 1000, null_frac),
             pick(specials, n_in, seed + 13)]
    return outer, inner


def unique_inner(inner, seed):
    """inner with its key column made unique (NULLs kept) — for single joins that must not raise."""
    k, nl = inner[0]
    u = np.argsort(ku.rand_u64(len(k), seed)).astype(np.int64) - len(k) // 3
    return [(u, nl)] + list(inner[1:])


def mode_cases() -> List[dict]:
    out = []
    O, I = mixed_tables(12_000, 5_000, 4_000, 0.03, 11)
    for jt in (INNER, LEFT, RIGHT, SEMI, ANTI):
        out.append(case(f"plain-{JT_NAME[jt]}", spec(jt, [0], [0], [I64]), O, I, build_parts=3, probe_parts=3))
    # NOT IN: the anti operand on the key column and on a non-key column; builds of one and two columns
    out.append(case("notin-keyop", spec(ANTI, [0], [0], [I64], anti_operands=[0]), O, I))
    out.append(case("notin-nonkeyop", spec(ANTI, [0], [0], [I64], anti_operands=[2]), O, I, probe_parts=3))
    out.append(case("notin-two-ops", spec(ANTI, [0], [0], [I64], anti_operands=[1, 2]), O, I))
    k, _ = I[0]
    one_nonull = [(k, None)]
    one_null = [ku.with_nulls(k, 0.001, 5)]
    assert one_null[0][1].any()
    out.append(case("notin-1col-nonull", spec(ANTI, [0], [0], [I64], anti_operands=[0]), O, one_nonull))
    out.append(case("notin-1col-null", spec(ANTI, [0], [0], [I64], anti_operands=[0]), O, one_null, build_parts=3))
    # two build columns, the first holding NULLs: NOT IN still answers row by row
    two_null0 = [one_null[0], I[1]]
    out.append(case("notin-2col-null0", spec(ANTI, [0], [0], [I64], anti_operands=[0]), O, two_null0))
    out.append(case("notin-2col-null0-key1", spec(ANTI, [1], [1], [I32], anti_operands=[1]),
                    O, [one_null[0], (I[1][0], None)]))
    out.append(case("notexists-1col-null", spec(ANTI, [0], [0], [I64]), O, one_null))
    # single joins over a unique inner key: fine; over duplicates: MoreThanOneRow; duplicates a condition hides: fine
    U = unique_inner(I, 21)
    for jt in (INNER, LEFT, RIGHT):
        out.append(case(f"single-{JT_NAME[jt]}", spec(jt, [0], [0], [I64], max_one_row=True), O, U))
        out.append(case(f"single-dup-{JT_NAME[jt]}", spec(jt, [0], [0], [I64], max_one_row=True), O, I))
        hidden = single_hidden_tables(jt, 33)
        out.append(case(f"single-hidden-{JT_NAME[jt]}", hidden[0], hidden[1], hidden[2]))
    # cond_ne: 1..4 terms over INT32 / INT64 columns of both sides of the join row left || right (inner || outer for
    # RIGHT); the values occur in the data, and the condition columns carry NULLs
    for jt in (INNER, LEFT, RIGHT, SEMI, ANTI):
        last = (2, 999) if jt == RIGHT else (2, int(O[2][0][5]))
        terms = [(1, 3), (5, 2), (4, int(O[0][0][7])), last]
        for nterm in (1, 2, 3, 4):
            out.append(case(f"cond{nterm}-{JT_NAME[jt]}", spec(jt, [0], [0], [I64], cond_ne=tuple(terms[:nterm])),
                            O, I, probe_parts=2))
    out.append(case("cond-notin", spec(ANTI, [0], [0], [I64], anti_operands=[2], cond_ne=((5, 2),)), O, I))
    for jt in (INNER, LEFT, RIGHT):
        out.append(case(f"build-outer-{JT_NAME[jt]}", spec(jt, [0], [0], [I64], build_outer=True), O, I,
                        build_parts=3, probe_parts=3))
    return out


def single_hidden_tables(jt, seed):
    """Every inner key has two rows, one of which the condition rejects (inner column 1 == -1): a single join whose
    second key match never passes."""
    n = 2000
    inner = [(np.repeat(np.arange(n, dtype=np.int64), 2), None), (np.tile(np.array([5, -1], np.int32), n), None),
             rcol(2 * n, seed, np.int32, 100, 0.1)]
    outer = [rcol(3000, seed + 1, np.int64, n + 500, 0.02), rcol(3000, seed + 2, np.int32, 9, 0.05)]
    flag_col = 1 if jt == RIGHT else len(outer) + 1
    return spec(jt, [0], [0], [I64], max_one_row=True, cond_ne=((flag_col, -1),)), outer, inner


# ---------------------------------------------------------------------------------------------- keys
def key_cases() -> List[dict]:
    out = []
    n_out, n_in = 12_000, 5_000
    # widening: (outer column type, inner column type, unified type)
    widen = [(np.int32, np.int32, I32), (np.int32, np.int64, I64), (np.int64, np.int32, I64), (np.int64, np.int64, I64),
             (np.int32, np.float64, F64), (np.int64, np.float64, F64), (np.float64, np.int32, F64),
             (np.float64, np.float64, F64), (np.int32, np.int32, I64), (np.int32, np.int32, F64)]
    for i, (to, ti, ut) in enumerate(widen):
        ok = rcol(n_out, 100 + i, np.int64, 3000, 0.02, -1500)
        ik = rcol(n_in, 200 + i, np.int64, 3000, 0.02, -1500)
        outer = [(ok[0].astype(to), ok[1]), rcol(n_out, 300 + i, np.int32, 50)]
        inner = [(ik[0].astype(ti), ik[1]), rcol(n_in, 400 + i, np.int64, 1 << 50)]
        tn = {np.int32: "i32", np.int64: "i64", np.float64: "f64"}
        for jt in (INNER, LEFT, ANTI):
            out.append(case(f"widen-{tn[to]}-{tn[ti]}-as-{['i32', 'i64', 'f64'][ut]}-{JT_NAME[jt]}",
                            spec(jt, [0], [0], [ut]), outer, inner))
    # BIGINT above 2^53 unified to DOUBLE: distinct BIGINTs that round to one double join each other
    base = 1 << 53
    big = np.array([base, base + 1, base + 2, base + 3, base + 4, -base - 1, -base - 2, INT64_MAX, INT64_MIN,
                    (1 << 62) + 1, (1 << 62) + 512], dtype=np.int64)
    outer = [pick(big, 3000, 41, 0.05), rcol(3000, 42, np.int32, 100)]
    inner = [pick(big, 500, 43, 0.05), rcol(500, 44, np.int32, 100)]
    inner_f = [(inner[0][0].astype(np.float64), inner[0][1]), inner[1]]
    for jt in (INNER, LEFT, SEMI, ANTI):
        out.append(case(f"bigint-as-double-{JT_NAME[jt]}", spec(jt, [0], [0], [F64]), outer, inner))
        out.append(case(f"bigint-vs-double-{JT_NAME[jt]}", spec(jt, [0], [0], [F64]), outer, inner_f))
        out.append(case(f"bigint-exact-{JT_NAME[jt]}", spec(jt, [0], [0], [I64]), outer, inner))
    # DOUBLE specials without signed zeros (the oracle agrees); NaN payloads never match
    specials = f64_array(FINITE_SPECIALS + NANS + [POS_ZERO])
    outer = [pick(specials, 4000, 51, 0.03), rcol(4000, 52, np.int32, 1000), pick(specials, 4000, 53)]
    inner = [pick(specials, 300, 54, 0.03), pick(specials, 300, 55), rcol(300, 56, np.int64, 1000)]
    for jt in (INNER, LEFT, RIGHT, SEMI, ANTI):
        out.append(case(f"double-specials-{JT_NAME[jt]}", spec(jt, [0], [0], [F64]), outer, inner))
    out.append(case("double-specials-notin", spec(ANTI, [0], [0], [F64], anti_operands=[0]), outer, inner))
    # ... and with both zeros: -0.0 joins only -0.0 (the oracle's answer depends on its bucket count here)
    zs = f64_array(FINITE_SPECIALS + NANS + [POS_ZERO, NEG_ZERO])
    outer = [pick(zs, 4000, 61, 0.03), rcol(4000, 62, np.int32, 1000)]
    inner = [pick(zs, 300, 63, 0.03), rcol(300, 64, np.int64, 1000)]
    for jt in (INNER, LEFT, RIGHT, SEMI, ANTI):
        out.append(case(f"double-signed-zero-{JT_NAME[jt]}", spec(jt, [0], [0], [F64]), outer, inner, oracle=False))
    # composite key with a signed-zero DOUBLE component
    ints = np.arange(4, dtype=np.int32)
    outer = [pick(zs, 4000, 65), pick(ints, 4000, 66), rcol(4000, 67, np.int32, 99)]
    inner = [pick(zs, 400, 68), pick(ints, 400, 69), rcol(400, 70, np.int64, 99)]
    out.append(case("double-signed-zero-2key", spec(INNER, [0, 1], [0, 1], [F64, I32]), outer, inner, oracle=False))
    # integer extremes: INT64_MIN is the generic table's empty-slot marker and has a slot of its own
    ext64 = np.array([INT64_MIN, INT64_MAX, INT32_MIN, INT32_MAX, -1, 0, 1, INT64_MIN + 1, INT64_MAX - 1], np.int64)
    ext32 = np.array([INT32_MIN, INT32_MAX, -1, 0, 1, INT32_MIN + 1], np.int32)
    for name, vals, kt in (("i64", ext64, I64), ("i32", ext32, I32)):
        outer = [pick(vals, 3000, 71, 0.02), rcol(3000, 72, np.int32, 1000)]
        inner_dup = [pick(vals, 200, 73, 0.02), rcol(200, 74, np.int64, 1000)]
        inner_uni = [(vals.copy(), None), rcol(len(vals), 75, np.int64, 1000)]
        for jt in (INNER, LEFT, RIGHT, SEMI, ANTI):
            out.append(case(f"extremes-{name}-dup-{JT_NAME[jt]}", spec(jt, [0], [0], [kt]), outer, inner_dup))
            out.append(case(f"extremes-{name}-unique-{JT_NAME[jt]}", spec(jt, [0], [0], [kt]), outer, inner_uni))
    # 1, 2, 3 and 8 keys over mixed types; outer tuples that differ from an inner tuple in exactly one component
    for nk in (1, 2, 3, 8):
        out.append(multi_key_case(nk, 80 + nk))
    out.append(digest_collision_case())
    return out


def multi_key_case(nk: int, seed: int) -> dict:
    types = [np.int64, np.int32, np.float64, np.int64, np.int32, np.float64, np.int64, np.int32][:nk]
    utypes = [I64, I32, F64, F64, I64, F64, I64, I32][:nk]
    n_in, n_out = 3000, 9000
    mod = max(3, round(n_in ** (1 / nk)))  # tuples repeat, but not thousands of times
    inner = []
    for c, t in enumerate(types):
        v = (ku.rand_u64(n_in, seed * 100 + c) % np.uint64(mod)).astype(np.int64) - mod // 2
        inner.append(ku.with_nulls(v.astype(t), 0.01, seed * 100 + 50 + c))
    # outer: copies of inner tuples, a third of them with one component moved off by one
    src = (ku.rand_u64(n_out, seed + 1) % np.uint64(n_in)).astype(np.int64)
    which = (ku.rand_u64(n_out, seed + 2) % np.uint64(nk)).astype(np.int64)
    moved = (ku.rand_u64(n_out, seed + 3) % np.uint64(3)) == 0
    outer = []
    for c, t in enumerate(types):
        d, nl = inner[c]
        v = d[src].copy()
        bump = moved & (which == c)
        v[bump] = v[bump] + t(1)
        outer.append((v, None if nl is None else nl[src]))
    outer.append(rcol(n_out, seed + 4, np.int32, 1000))
    inner.append(rcol(n_in, seed + 5, np.int64, 1000))
    keys = list(range(nk))
    return case(f"keys{nk}", spec(LEFT, keys, keys, utypes), outer, inner, probe_parts=2)


# ---- digest collisions: a restatement of join.cu's composite-key digest, used to build tuples whose digests are equal
_M64 = 2**64 - 1
_C1, _C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53


def _fmix64(x: int) -> int:
    x ^= x >> 33
    x = (x * _C1) & _M64
    x ^= x >> 33
    x = (x * _C2) & _M64
    return x ^ (x >> 33)


def _fmix64_inv(x: int) -> int:
    x ^= x >> 33
    x = (x * pow(_C2, -1, 2**64)) & _M64
    x ^= x >> 33
    x = (x * pow(_C1, -1, 2**64)) & _M64
    return x ^ (x >> 33)


def _digest_prefix(keys: List[int]) -> int:
    h = 0x243F6A8885A308D3
    for c, k in enumerate(keys):
        h = (_fmix64(h ^ (k & _M64)) + 0x9E3779B97F4A7C15 * (c + 1)) & _M64
    return h


def _last_key_for(prefix: List[int], digest: int) -> int:
    """The last BIGINT component that gives the tuple prefix + [k] the pre-fold digest `digest`."""
    c = len(prefix)
    k = _fmix64_inv((digest - 0x9E3779B97F4A7C15 * (c + 1)) & _M64) ^ _digest_prefix(prefix)
    return k - 2**64 if k >= 2**63 else k


def digest_collision_case() -> dict:
    """Composite BIGINT keys whose 64-bit digests are equal, so one table slot holds unequal tuples and only the key
    verification tells them apart:
      * a digest equal to the empty-slot marker is folded onto marker ^ 1, so (a, x) and (a, y) with those two digests
        share a slot while differing in the last component only;
      * (b, z) is solved to have the digest of (a, x) with b != a: a full 64-bit collision of two different tuples."""
    marker = 2**63
    inner_rows, outer_rows = [], []
    for a in range(1, 41):
        x = _last_key_for([a], marker)
        y = _last_key_for([a], marker ^ 1)
        inner_rows += [(a, x)]
        outer_rows += [(a, y), (a, x)]
        b = a + 1000
        z = _last_key_for([b], _digest_prefix([a, x]))
        assert _digest_prefix([b, z]) == _digest_prefix([a, x])
        inner_rows += [(b, z), (a, y + 1)]
        outer_rows += [(b, x), (a, z), (b, z)]
    ik = np.array(inner_rows, dtype=np.int64)
    ok = np.array(outer_rows, dtype=np.int64)
    inner = [(ik[:, 0].copy(), None), (ik[:, 1].copy(), None), (np.arange(len(ik), dtype=np.int32), None)]
    outer = [(ok[:, 0].copy(), None), (ok[:, 1].copy(), None), (np.arange(len(ok), dtype=np.int64), None)]
    return case("digest-collisions", spec(LEFT, [0, 1], [0, 1], [I64, I64]), outer, inner)


# ---------------------------------------------------------------------------------------------- build shapes
def shape_cases() -> List[dict]:
    out = []
    n_out = 12_000
    for nb in (0, 1, 8192, 8193, 200_003):
        O, I = mixed_tables(n_out, nb, max(nb, 1), 0.0, 500 + nb % 97)
        I = [(np.argsort(ku.rand_u64(nb, 7)).astype(np.int64) - nb // 3, None)] + I[1:] if nb else I  # unique keys
        parts = 7 if nb > 7 else 1
        for jt in (INNER, LEFT, RIGHT, SEMI, ANTI):
            out.append(case(f"build{nb}-unique-{JT_NAME[jt]}", spec(jt, [0], [0], [I64]), O, I,
                            build_parts=parts, probe_parts=3))
        out.append(case(f"build{nb}-unique-notin", spec(ANTI, [0], [0], [I64], anti_operands=[0]), O, I))
    O, I = mixed_tables(300, 8193, 40, 0.01, 601)    # ~200 inner rows per key
    for jt in (INNER, LEFT, SEMI, ANTI):
        out.append(case(f"heavy-dups-{JT_NAME[jt]}", spec(jt, [0], [0], [I64]), O, I, build_parts=3))
    O, I = mixed_tables(300, 500, 1, 0.0, 602)    # one key value: every match walks one 500-row chain
    I[0] = (np.full(500, 7, np.int64), None)
    O[0] = (np.where(np.arange(300) % 3 == 0, O[0][0], 7).astype(np.int64), None)
    for jt in (INNER, RIGHT, SEMI, ANTI):
        out.append(case(f"one-key-{JT_NAME[jt]}", spec(jt, [0], [0], [I64]), O, I))
    O, I = mixed_tables(n_out, 5_000, 100, 0.02, 603)
    I[0] = (I[0][0], np.ones(5_000, bool))       # all-NULL key column: nothing is inserted
    for jt in (INNER, LEFT, RIGHT, SEMI, ANTI):
        out.append(case(f"null-keys-{JT_NAME[jt]}", spec(jt, [0], [0], [I64]), O, I, build_parts=3))
    out.append(case("null-keys-notin", spec(ANTI, [0], [0], [I64], anti_operands=[0]), O, I[:1]))
    return out


# ---------------------------------------------------------------------------------------------- batching
def batching_cases() -> List[dict]:
    """The build side in 1, 3 or 7 batches where only some batches carry a NULL mask (the GPU run passes a mask only
    for a batch that holds a NULL), including a mask that first appears on the last batch."""
    out = []
    n_in = 7_000
    O, I = mixed_tables(20_000, n_in, 2_500, 0.0, 701)
    for parts in (1, 3, 7):
        for where in (("last",) if parts == 1 else ("last", "middle", "first")):
            edges = np.linspace(0, n_in, parts + 1).astype(int)
            b = {"last": parts - 1, "middle": parts // 2, "first": 0}[where]
            lo, hi = edges[b], edges[b + 1]
            m0, m2 = np.zeros(n_in, bool), np.zeros(n_in, bool)
            m0[lo:hi] = (ku.rand_u64(hi - lo, 702 + parts) % np.uint64(10)) == 0
            m2[lo:hi] = (ku.rand_u64(hi - lo, 703 + parts) % np.uint64(10)) == 0
            Ib = [(I[0][0], m0), (I[1][0], None), (I[2][0], m2), I[3]]
            for jt in (INNER, LEFT, ANTI):
                out.append(case(f"masks-{where}-of-{parts}-{JT_NAME[jt]}", spec(jt, [0], [0], [I64]), O, Ib,
                                build_parts=parts, probe_parts=3))
            out.append(case(f"masks-{where}-of-{parts}-notin1", spec(ANTI, [0], [0], [I64], anti_operands=[0]),
                            O, Ib[:1], build_parts=parts))
    return out


def all_cases() -> List[dict]:
    return mode_cases() + key_cases() + shape_cases() + batching_cases()


def cases_by_id() -> dict:
    cs = all_cases()
    d = {c["id"]: c for c in cs}
    assert len(d) == len(cs), "duplicate case ids"
    return d
