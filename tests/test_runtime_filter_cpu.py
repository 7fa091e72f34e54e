"""CPU checks of the runtime bloom filter's contract: the numpy restatement (tests/bloom_ref.py) against published and
libxxhash XXH64 vectors, the reference's put64 positions and filter sizing worked by hand, the product's
api.bloom_sizing against the restatement, and the C-ABI / JNI declarations of the six gsql_bloom_* entry points."""
import json
import os
import struct

import numpy as np
import pytest

from tests import bloom_ref as br
from tests import kat_util as ku

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "xxh64_long.json")


def _golden():
    with open(GOLDEN) as fh:
        return json.load(fh)


def test_xxh64_matches_the_published_and_libxxhash_vectors():
    g = _golden()
    assert br.xxh64_short(b"") == int(g["published"]["empty_string"], 16) == 0xEF46DB3751D8E999
    vals = np.array([v for v, _ in g["long"]], dtype=np.int64)
    exp = np.array([int(h, 16) for _, h in g["long"]], dtype=np.uint64)
    assert len(vals) == 1000
    assert np.array_equal(br.xxh64_long(vals), exp)
    # the scalar specification path (8-byte lane, then the avalanche) agrees with the vectorised one
    for v, h in g["long"][:50]:
        assert br.xxh64_short(struct.pack("<q", v)) == int(h, 16)
    # the values the issue worked by hand
    assert [int(x) for x in br.xxh64_long([0, 1, -1, 42])] == [0x34C96ACDCADB1BBB, 0x9F29CB17A2A49995, 0x85D136ADB773C6C9,
                                                              0xB556806FB6D14353]


def test_xxh64_matches_libxxhash_on_random_longs():
    xxhash = pytest.importorskip("xxhash")
    vals = ku.rand_u64(100_000, 4242).view(np.int64)
    exp = np.array([xxhash.xxh64_intdigest(struct.pack("<q", int(v))) for v in vals], dtype=np.uint64)
    assert np.array_equal(br.xxh64_long(vals), exp)


def test_xxh64_inverse_round_trips():
    for h in [0, 1, (1 << 64) - 1, 0x7FFFFFFF, 0x8000000000000000] + [int(x) for x in ku.rand_u64(200, 7)]:
        v = br.xxh64_long_inverse(h)
        assert int(br.xxh64_long([v])[0]) == h


def test_key_longs_follow_the_blocks_hasher_input():
    i32 = np.array([-1, 5, -(1 << 31)], dtype=np.int32)
    assert br.key_longs(i32).tolist() == [-1, 5, -(1 << 31)]                      # putInt -> putLong sign-extends
    d = np.array([-0.0, 0.0, float("nan")], dtype=np.float64)
    bits = br.key_longs(d).view(np.uint64).tolist()
    assert bits[0] == 1 << 63 and bits[1] == 0 and bits[2] == struct.unpack("<Q", struct.pack("<d", float("nan")))[0]
    payload = np.array([0x7FF8000000000001, 0x7FF0000000000001], dtype=np.int64).view(np.float64)
    assert br.key_longs(payload).tolist() == [0x7FF8000000000001, 0x7FF0000000000001]  # raw bits: NaN payloads kept
    assert br.key_longs(np.array([7, 8], np.int64), np.array([True, False])).tolist() == [0, 8]   # NULL -> NULL_VALUE 0


def test_sizing_matches_the_hand_worked_values():
    assert br.DEFAULT_FPP == 0.029999999329447746 != 0.03                         # 0.03f widened to double
    assert br.create_empty_sizing(1000, br.DEFAULT_FPP) == (7360, 5)
    assert br.create_empty_sizing(2 * 1024 * 1024, br.DEFAULT_FPP) == (15_305_984, 5)
    assert br.create_empty_sizing(1, br.DEFAULT_FPP) == (64, 44)
    assert br.sizing(1000) == br.sizing(10) == br.sizing(0) == (7360, 5)          # clamped up to BLOOM_FILTER_MIN_SIZE
    assert br.sizing(2 * 1024 * 1024) == (15_305_984, 5)
    # above BLOOM_FILTER_MAX_SIZE the size is clamped and findMinFpp raises the fpp: the filter shrinks
    big = 50_000_000
    assert br.sizing(big) == br.create_empty_sizing(2 * 1024 * 1024, np.exp(-3.843 * 2 * 1024 * 1024 / big)) == (703_616, 1)
    # the 0.03f quirk is observable: at some sizes a double 0.03 would give a filter one word smaller
    assert br.sizing(34_506) == br.create_empty_sizing(34_506, br.DEFAULT_FPP) == (251_904, 5)
    assert br.create_empty_sizing(34_506, 0.03) == (251_840, 5)
    # findMinFpp: a filter much larger than ndv gets a lower fpp than DEFAULT_FPP
    nb, k = br.sizing(100, min_size=1000)
    assert (nb, k) == br.create_empty_sizing(1000, max(np.exp(-3.843 * 1000 / 100), br.DEFAULT_FPP))


def test_put64_positions_match_the_hand_worked_values():
    h = br.xxh64_long([42, 0])
    pos = br.positions(h, 7360, 5)
    assert pos[0].tolist() == [3586, 1841, 5024, 3279, 6462]
    assert pos[1].tolist() == [1096, 4757, 5986, 2287, 3516]
    # a NULL key sets what key 0 sets
    w_null = br.build([(np.array([123], np.int64), np.array([True]))], 0, 7360, 5)
    w_zero = br.build([(np.array([0], np.int64), None)], 0, 7360, 5)
    assert np.array_equal(w_null, w_zero)
    assert sum(bin(int(x)).count("1") for x in w_zero) == 5
    # bit i lives in word i >> 6 at bit i & 63 (BitSet.java)
    assert all((int(w_zero[p >> 6]) >> (p & 63)) & 1 for p in pos[1].tolist())


def test_put64_clears_the_sign_bit_like_java_int_arithmetic():
    """combined = hash1 + hash2 wraps as a Java int; a negative combined has its sign bit cleared before the modulo."""
    def java_positions(h, nbits, k):
        def to_int(x):
            x &= 0xFFFFFFFF
            return x - (1 << 32) if x >> 31 else x
        h1, h2 = to_int(h), to_int(h >> 32)
        c, out = to_int(h1 + h2), []
        for _ in range(k):
            if c < 0:
                c &= 0x7FFFFFFF
            out.append(c % nbits)
            c = to_int(c + h2)
        return out
    hs = [int(x) for x in ku.rand_u64(2000, 99)] + [0xFFFFFFFF_FFFFFFFF, 0x80000000_80000000, 0x7FFFFFFF_00000000, 0x00000001_7FFFFFFF]
    for nbits, k in [(64, 44), (7360, 5), (br.MAX_BITS, 3)]:
        got = br.positions(np.array(hs, dtype=np.uint64), nbits, k)
        for h, row in zip(hs, got):
            assert row.tolist() == java_positions(h, nbits, k)


def test_fastmod_is_exact_at_the_extremes():
    for d in [64, 128, 7360, 15_305_984, (1 << 31) - 128, br.MAX_BITS]:
        for a in [0, 1, d - 1, d, d + 1, (1 << 31) - 2, (1 << 31) - 1] + [int(x) for x in ku.rand_u64(500, d) % np.uint64(1 << 31)]:
            assert br.fastmod_u32(a, d) == a % d, (a, d)


def test_might_contain_accepts_every_built_key():
    keys = (ku.rand_u64(5000, 3) % np.uint64(1 << 40)).astype(np.int64)
    nb, k = br.sizing(5000)
    w = br.build([(keys, None)], 0, nb, k)
    assert br.might_contain(w, keys, None, k).all()
    other = (ku.rand_u64(20000, 4) % np.uint64(1 << 40)).astype(np.int64) + (1 << 41)
    fp = br.might_contain(w, other, None, k).mean()
    assert 0 < fp < 0.05


@pytest.mark.parametrize("ndv", [-5, 0, 1, 999, 1000, 1001, 12_345, 34_506, 300_000, 2 * 1024 * 1024, 2 * 1024 * 1024 + 1, 10**9])
def test_api_bloom_sizing_equals_the_restatement(ndv):
    from galaxysql_b200 import api
    assert api.bloom_sizing(ndv) == br.sizing(ndv)
    assert api.bloom_sizing(ndv, min_size=1, max_size=1 << 16) == br.sizing(ndv, min_size=1, max_size=1 << 16)


def test_abi_declares_the_bloom_entry_points():
    from galaxysql_b200 import native as N
    for name in ("gsql_bloom_create", "gsql_bloom_put", "gsql_bloom_merge", "gsql_bloom_bitmap", "gsql_bloom_filter", "gsql_bloom_destroy"):
        assert name in N.ABI_SYMBOLS
    src = open(os.path.join(ROOT, "include", "gsql_gpu.h")).read()
    assert "#define GSQL_ABI_VERSION 1" in src
    assert "typedef struct gsql_bloom gsql_bloom;" in src


def test_jni_declares_the_bloom_natives():
    src = open(os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor", "operator", "gpu", "GpuNative.java")).read()
    shim = open(os.path.join(ROOT, "jni", "gsql_jni.c")).read()
    for name in ("bloomCreate", "bloomPut", "bloomMerge", "bloomBitmapOr", "bloomFilter", "bloomDestroy"):
        assert f" {name}(" in src, name
        assert f"NATIVE(" in shim and f", {name})" in shim, name


_JNI_HARNESS = r'''
#include <stdio.h>
#include <string.h>
#include "gsql_jni.c"

typedef struct { jsize len; } fake_array;
static int region_calls, critical_calls, throws;
static char last_msg[256];
static jclass find_class(JNIEnv *e, const char *n) { return (jclass)n; }
static jint throw_new(JNIEnv *e, jclass c, const char *m) { throws++; snprintf(last_msg, sizeof last_msg, "%s", m); return 0; }
static jboolean exception_check(JNIEnv *e) { return 0; }
static jsize array_length(JNIEnv *e, jarray a) { return ((fake_array *)a)->len; }
static void long_region(JNIEnv *e, jlongArray a, jsize s, jsize n, jlong *b) { region_calls++; memset(b, 0, (size_t)n * 8); }
static void *critical(JNIEnv *e, jarray a, jboolean *c) { critical_calls++; return NULL; }
static void release_critical(JNIEnv *e, jarray a, void *p, jint m) {}

int main(void) {
    struct JNINativeInterface_ fns;
    memset(&fns, 0, sizeof fns);
    fns.FindClass = find_class; fns.ThrowNew = throw_new; fns.ExceptionCheck = exception_check;
    fns.GetArrayLength = array_length; fns.GetLongArrayRegion = long_region;
    fns.GetPrimitiveArrayCritical = critical; fns.ReleasePrimitiveArrayCritical = release_critical;
    const struct JNINativeInterface_ *tbl = &fns;
    JNIEnv *env = (JNIEnv *)&tbl;
    jbloom h = {NULL, NULL, 115};                 /* a 7360-bit filter: 115 words */
    jlong bh = (jlong)(intptr_t)&h;
    fake_array shorter = {114}, exact = {115}, longer = {116}, two = {230};
    /* bitmap-or: null, shorter and longer arrays are rejected before anything is copied */
    Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_bloomBitmapOr(env, NULL, bh, NULL);
    printf("or_null %d %d %s\n", throws, critical_calls, last_msg);
    Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_bloomBitmapOr(env, NULL, bh, &shorter);
    printf("or_short %d %d %s\n", throws, critical_calls, last_msg);
    Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_bloomBitmapOr(env, NULL, bh, &longer);
    printf("or_long %d %d %s\n", throws, critical_calls, last_msg);
    /* merge: words.length must be nfilters * nwords */
    Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_bloomMerge(env, NULL, bh, NULL, 1);
    printf("merge_null %d %d %s\n", throws, region_calls, last_msg);
    Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_bloomMerge(env, NULL, bh, &exact, 2);
    printf("merge_short %d %d %s\n", throws, region_calls, last_msg);
    Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_bloomMerge(env, NULL, bh, &two, 1);
    printf("merge_long %d %d %s\n", throws, region_calls, last_msg);
    Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_bloomMerge(env, NULL, bh, &exact, 0);
    printf("merge_zero %d %d %s\n", throws, region_calls, last_msg);
    /* the right size passes the check (the library then rejects the fake handle, or host memory is unavailable) */
    last_msg[0] = 0;
    Java_com_alibaba_polardbx_executor_operator_gpu_GpuNative_bloomMerge(env, NULL, bh, &two, 2);
    printf("merge_ok %s\n", last_msg);
    return 0;
}
'''


def test_jni_bloom_natives_reject_arrays_of_the_wrong_size():
    """bloomBitmapOr / bloomMerge check the Java long[] against the filter's size before copying a byte: a getBitmap() array
    of another filter, or null, becomes a GpuExecutorException instead of a heap overflow or over-read.  Runs the shim's
    natives against a fake JNIEnv."""
    import subprocess
    import tempfile
    import __graft_entry__ as g
    g.build()
    so_dir = os.path.join(ROOT, "galaxysql_b200", "_build")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "h.c"), "w").write(_JNI_HARNESS)
        exe = os.path.join(d, "h")
        subprocess.check_call(["gcc", "-Wall", "-Werror", "-Wno-unused-function", "-I", os.path.join(ROOT, "jni", "stub"), "-I",
                               os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "jni"), os.path.join(d, "h.c"), "-L", so_dir,
                               "-lgsql_gpu", f"-Wl,-rpath,{so_dir}", "-o", exe])
        out = dict(line.split(" ", 1) for line in subprocess.check_output([exe], text=True).splitlines())
    size_msg = "must hold"
    for i, case in enumerate(["or_null", "or_short", "or_long"]):
        throws, critical, msg = out[case].split(" ", 2)
        assert int(throws) == i + 1 and int(critical) == 0 and "bloomBitmapOr" in msg and size_msg in msg, (case, out[case])
    for i, case in enumerate(["merge_null", "merge_short", "merge_long", "merge_zero"]):
        throws, region, msg = out[case].split(" ", 2)
        assert int(throws) == i + 4 and int(region) == 0 and "bloomMerge" in msg and size_msg in msg, (case, out[case])
    assert size_msg not in out.get("merge_ok", "")


def test_java_runtime_filter_operators_use_the_natives_as_documented():
    """The build-side operator ORs the GPU bitmap into the shared filter under its lock and only then closes the
    BloomFilterProduce (whose last closer sends the bitmaps); the probe-side operator loads each arrived bitmap into an
    empty GPU filter of its size; the factory keeps the stock operator when GpuSupport says no."""
    base = os.path.join(ROOT, "java", "com", "alibaba", "polardbx", "executor")
    build = open(os.path.join(base, "operator", "GpuRuntimeFilterBuilderExec.java")).read()
    i_or, i_close = build.index("GpuNative.bloomBitmapOr(blooms[i], bf.getBitmap())"), build.index("filterClient.close()")
    assert "synchronized (bf)" in build[:i_or] and i_or < i_close
    apply = open(os.path.join(base, "operator", "GpuRuntimeFilterExec.java")).read()
    assert "GpuNative.bloomCreate(ctx, words.length * (long) Long.SIZE, bf.getNumHashFunctions())" in apply
    assert "GpuNative.bloomMerge(blooms[i], words, 1)" in apply
    factory = open(os.path.join(base, "mpp", "operator", "factory", "GpuRuntimeFilterBuilderExecFactory.java")).read()
    assert "GpuSupport.runtimeFilterSupported(" in factory and "new RuntimeFilterBuilderExec(" in factory
