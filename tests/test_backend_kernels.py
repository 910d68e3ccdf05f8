"""GPU tier: the CUDA backend's own primitives (csrc/gar_engine.cu), one at a time, against exact numpy references.

The host simulation runs a serial loop in place of each of these, so whole-diff parity only reaches them at the shapes a model
happens to produce.  Here tests/cuda/backend_harness.cu calls each member of the engine on host arrays:
  * exclusive_scan    decoupled look-back over 2048-item tiles, uint4 fast path and scalar tail
  * sort_pairs        stable 8-bit LSD radix passes, odd pass counts copied back
  * for_each_multi    several functors' block ranges in one launch
  * for_each_dyn / for_each_warp_dyn   counts that live on the device, clamped to a capacity, whole warps
  * fill32            memset path for 0, a capped grid-stride kernel otherwise
  * for_each_staged   TMA bulk copy of a block's string window into shared memory, and the view that picks shared memory
                      or the slab per string
Every comparison is integer and bit-exact.  The staged row passes of the real pipeline and the GAR_NO_TMA / GAR_TMA_ALL
switches are checked end to end against the oracle at the bottom of the file."""
import ctypes as C
import importlib
import os

import numpy as np
import pytest

import randmodel

pytestmark = pytest.mark.gpu

OFF_MASK = (1 << 40) - 1
_u32p, _u8p, _u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)


class Harness:
    def __init__(self, path):
        lib = self.lib = C.CDLL(str(path))
        lib.bh_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        lib.bh_destroy.argtypes = [C.c_void_p]
        lib.bh_error.argtypes = [C.c_void_p]
        lib.bh_error.restype = C.c_char_p
        lib.bh_exclusive_scan.argtypes = [C.c_void_p, _u32p, C.c_uint32]
        lib.bh_sort_pairs.argtypes = [C.c_void_p, _u32p, _u32p, C.c_uint32, C.c_int]
        lib.bh_for_each_multi.argtypes = [C.c_void_p, _u32p, C.c_int, _u32p, _u32p]
        lib.bh_for_each_dyn.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32, _u32p, _u8p, _u32p, _u32p]
        lib.bh_fill32.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, _u32p]
        lib.bh_for_each_staged.argtypes = [C.c_void_p, C.c_int, _u64p, C.c_uint32, _u8p, C.c_uint64, C.c_uint32, _u8p, C.c_uint64, C.c_uint32,
                                           _u8p, _u64p, C.c_uint64, _u8p, _u8p]
        self.h = C.c_void_p()
        rc = lib.bh_create(0, C.byref(self.h))
        assert rc == 0, lib.bh_error(None).decode()

    def _ok(self, rc):
        assert rc == 0, self.lib.bh_error(self.h).decode()

    def scan(self, x):
        d = np.ascontiguousarray(x, dtype=np.uint32).copy()
        self._ok(self.lib.bh_exclusive_scan(self.h, d.ctypes.data_as(_u32p), len(d)))
        return d

    def sort_pairs(self, keys, vals, bits):
        k = np.ascontiguousarray(keys, dtype=np.uint32).copy()
        v = np.ascontiguousarray(vals, dtype=np.uint32).copy()
        self._ok(self.lib.bh_sort_pairs(self.h, k.ctypes.data_as(_u32p), v.ctypes.data_as(_u32p), len(k), bits))
        return k, v

    def multi(self, ns):
        ns = np.asarray(ns, dtype=np.uint32)
        hits = np.zeros(max(1, int(ns.sum())), dtype=np.uint32)
        stray = np.zeros(1, dtype=np.uint32)
        self._ok(self.lib.bh_for_each_multi(self.h, ns.ctypes.data_as(_u32p), len(ns), hits.ctypes.data_as(_u32p), stray.ctypes.data_as(_u32p)))
        return hits[:int(ns.sum())], int(stray[0])

    def dyn(self, warp, n, cap):
        length = (cap + 255) // 256 * 256
        hits = np.zeros(length, dtype=np.uint32)
        valid = np.zeros(length, dtype=np.uint8)
        stray, partial = np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint32)
        self._ok(self.lib.bh_for_each_dyn(self.h, int(warp), n, cap, hits.ctypes.data_as(_u32p), valid.ctypes.data_as(_u8p), stray.ctypes.data_as(_u32p),
                                          partial.ctypes.data_as(_u32p)))
        return hits, valid, int(stray[0]), int(partial[0])

    def fill32(self, v, n, tail, sentinel):
        out = np.zeros(n + tail, dtype=np.uint32)
        self._ok(self.lib.bh_fill32(self.h, v, n, tail, sentinel, out.ctypes.data_as(_u32p)))
        return out

    def staged(self, variant, refs, slabs, shifts, no_window):
        refs = np.ascontiguousarray(refs, dtype=np.uint64)  # [n, 2]
        n = refs.shape[0]
        lens = (refs >> np.uint64(40)).astype(np.uint64).reshape(-1)
        begin = np.zeros(2 * n, dtype=np.uint64)
        begin[1:] = np.cumsum(lens)[:-1]
        out_len = int(lens.sum())
        out = np.zeros(max(1, out_len), dtype=np.uint8)
        flags = np.zeros(2 * n, dtype=np.uint8)
        s0, s1 = (np.frombuffer(bytes(s), dtype=np.uint8).copy() for s in slabs)
        nw = np.ascontiguousarray(no_window, dtype=np.uint8)
        self._ok(self.lib.bh_for_each_staged(self.h, variant, refs.ctypes.data_as(_u64p), n, s0.ctypes.data_as(_u8p), len(s0), shifts[0],
                                             s1.ctypes.data_as(_u8p), len(s1), shifts[1], nw.ctypes.data_as(_u8p), begin.ctypes.data_as(_u64p),
                                             out_len, out.ctypes.data_as(_u8p), flags.ctypes.data_as(_u8p)))
        return out, begin, flags.reshape(n, 2)

    def close(self):
        if self.h:
            self.lib.bh_destroy(self.h)
            self.h = C.c_void_p()


@pytest.fixture(scope="module")
def harness():
    import __graft_entry__ as ge
    h = Harness(ge.build_backend_harness())
    yield h
    h.close()


# ------------------------------------------------------------------ exclusive scan

SCAN_SIZES = [1, 7, 8, 9, 2047, 2048, 2049, 32 * 2048, 33 * 2048 + 1, 1000 * 2048 + 5, 2 ** 25 + 3]


def scan_ref(x):
    out = np.zeros(len(x), dtype=np.uint64)
    out[1:] = np.cumsum(x.astype(np.uint64))[:-1]
    return (out & 0xFFFFFFFF).astype(np.uint32)


@pytest.mark.parametrize("values", ["random", "zeros", "ones", "max"])
@pytest.mark.parametrize("n", SCAN_SIZES)
def test_exclusive_scan(harness, n, values):
    rng = np.random.default_rng(n)
    x = {"random": lambda: rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32), "zeros": lambda: np.zeros(n, np.uint32),
         "ones": lambda: np.ones(n, np.uint32), "max": lambda: np.full(n, 0xFFFFFFFF, np.uint32)}[values]()
    want = scan_ref(x)
    for run in range(2):  # the second run on the same engine starts from the tile states and ticket the first one left
        got = harness.scan(x)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (run, int(bad[0]), int(got[bad[0]]), int(want[bad[0]]))


# ------------------------------------------------------------------ radix sort

SORT_BITS = [1, 5, 8, 9, 16, 17, 24, 25, 32]
SORT_SIZES = [1, 255, 2047, 2048, 2049, 3 * 2048 + 17, 10 ** 6, 10 ** 7]


def sort_keys(rng, n, bits, dist):
    top = 1 << bits
    if dist == "uniform":
        return rng.integers(0, top, n, dtype=np.uint64).astype(np.uint32)
    if dist == "four":
        return rng.choice(rng.integers(0, top, 4, dtype=np.uint64), n).astype(np.uint32)
    if dist == "equal":
        return np.full(n, rng.integers(0, top), dtype=np.uint32)
    k = np.sort(rng.integers(0, top, n, dtype=np.uint64).astype(np.uint32))
    return k if dist == "sorted" else k[::-1].copy()


@pytest.mark.parametrize("dist", ["uniform", "four", "equal", "sorted", "reversed"])
@pytest.mark.parametrize("n", SORT_SIZES)
def test_sort_pairs_is_a_stable_sort(harness, n, dist):
    """vals = 0..n-1, so the values out are the stable permutation itself: any tie out of input order shows."""
    if n == 10 ** 7 and dist != "uniform":
        pytest.skip("10^7 keys run the uniform distribution only: the others are covered at 10^6, which already spans ~490 tiles")
    rng = np.random.default_rng(n * 7 + len(dist))
    vals = np.arange(n, dtype=np.uint32)
    for bits in SORT_BITS:
        keys = sort_keys(rng, n, bits, dist)
        perm = np.argsort(keys, kind="stable").astype(np.uint32)
        k, v = harness.sort_pairs(keys, vals, bits)
        assert np.array_equal(v, perm), (bits, int(np.flatnonzero(v != perm)[0]))
        assert np.array_equal(k, keys[perm]), bits


def test_sort_pairs_sorts_only_the_bits_it_is_given(harness):
    """The passes see the low 8 * ceil(bits / 8) bits: keys above them keep their input order (the host simulation sorts the
    same way, so a caller that passes too few bits fails there as well)."""
    rng = np.random.default_rng(5)
    n = 5000
    keys = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    for bits in (5, 9, 20):
        seen = 8 * ((bits + 7) // 8)
        perm = np.argsort(keys & np.uint32((1 << seen) - 1), kind="stable").astype(np.uint32)
        k, v = harness.sort_pairs(keys, np.arange(n, dtype=np.uint32), bits)
        assert np.array_equal(v, perm) and np.array_equal(k, keys[perm]), bits


# ------------------------------------------------------------------ fused and device-counted launches

def multi_cases():
    sizes = [0, 1, 255, 256, 257, 100_000]
    cases = [[0], [1], [100_000], [0, 0, 0], [0, 257], [257, 0], [1, 0, 255], [0, 256, 0, 0, 255, 100_000, 0, 257], [0] * 8, [257] * 8,
             [100_000, 1, 1, 1, 1, 1, 1, 0]]
    rng = np.random.default_rng(8)
    for k in range(1, 9):
        for _ in range(3):
            cases.append([int(x) for x in rng.choice(sizes, k)])
    return cases


@pytest.mark.parametrize("ns", multi_cases(), ids=lambda ns: "-".join(map(str, ns)))
def test_for_each_multi_visits_each_row_once(harness, ns):
    hits, stray = harness.multi(ns)
    assert stray == 0
    assert (hits == 1).all(), int(np.flatnonzero(hits != 1)[0])


DYN_CAPS = [1, 31, 32, 256, 1000]


def dyn_counts(cap):
    return sorted({0, 1, 31, 32, 33, cap - 1, cap, cap + 1, 10 * cap})


@pytest.mark.parametrize("cap", DYN_CAPS)
def test_for_each_dyn_clamps_to_the_capacity(harness, cap):
    for n in dyn_counts(cap):
        hits, _, stray, _ = harness.dyn(False, n, cap)
        m = min(n, cap)
        assert stray == 0
        assert (hits[:m] == 1).all() and (hits[m:] == 0).all(), (n, cap)


@pytest.mark.parametrize("cap", DYN_CAPS)
def test_for_each_warp_dyn_runs_whole_warps(harness, cap):
    for n in dyn_counts(cap):
        hits, valid, stray, partial = harness.dyn(True, n, cap)
        m = min(n, cap)
        r = (m + 31) // 32 * 32
        assert stray == 0 and partial == 0, (n, cap, stray, partial)
        assert (hits[:r] == 1).all() and (hits[r:] == 0).all(), (n, cap)
        assert np.array_equal(valid[:r], (np.arange(r) < m).astype(np.uint8)), (n, cap)


@pytest.mark.parametrize("v", [0, 7, 0xFFFFFFFF])
@pytest.mark.parametrize("n", [1, 255, 132 * 16 * 256 - 1, 132 * 16 * 256 + 1, 2 ** 25])
def test_fill32(harness, n, v):
    sentinel = 0xA5A5A5A5
    out = harness.fill32(v, n, 64, sentinel)
    assert (out[:n] == v).all(), int(np.flatnonzero(out[:n] != v)[0])
    assert (out[n:] == sentinel).all()


# ------------------------------------------------------------------ TMA-staged string windows

STAGE_VARIANTS = {0: (2, 1024), 1: (1, 24 * 1024), 2: (2, 16 * 1024)}  # harness variant -> (windows, bytes per window)


def staged_rule(o, ln, cap, window, aligned):
    """gar_engine.cu k_for_each_staged + StagedView for one block and window: which strings are read from shared memory."""
    o, ln = o.astype(np.int64), ln.astype(np.int64)
    lo, hi = int(o[0]), int(o[-1] + ln[-1])
    if not window or not aligned or hi <= lo:
        return np.zeros(len(o), dtype=bool)
    lo16 = lo & ~15
    span = min(((hi - lo16 + 15) & ~15) + 16, cap)
    return (o >= lo16) & (o + ln + 16 <= lo16 + span)


def block_refs(rng, case, cap, rows, slab_len):
    """String refs of one block whose window is `case` (rows > 2).  Besides the first and last row, which set the window, the block
    holds strings on both sides of every edge of the staged range: starting at lo16 - 1 and lo16, ending at (staged end) - 16
    (still staged) and - 15 (from the slab), empty strings at the same places, and random strings anywhere in the slab."""
    lo, hi = {"fits": (256, 256 + cap - 16), "over_by_1": (256, 256 + cap - 15), "unaligned_lo": (263, 263 + cap // 2), "small": (1000, 1100),
              "slab_end": (slab_len - cap // 2 - 3, slab_len), "reversed": (cap + 500, 300), "equal": (2000, 2000), "no_window": (512, 900),
              "wide": (48, 48 + 3 * cap)}[case]
    first_len = min(int(rng.integers(1, 40)), slab_len - lo) if case != "equal" else 0
    last_len = min(int(rng.integers(1, 40)), hi)
    o = rng.integers(0, slab_len - 64, rows).astype(np.int64)
    ln = rng.integers(0, 64, rows).astype(np.int64)
    lo16 = lo & ~15
    end = lo16 + min(((hi - lo16 + 15) & ~15) + 16, cap) if hi > lo else lo16
    probes = [(lo16, 10), (lo16 - 1, 10), (lo16, 0), (end - 16 - 9, 9), (end - 15 - 9, 9), (end - 16, 0), (end - 15, 0), (end - 17, 1)]
    slots = rng.choice(np.arange(1, rows - 1), len(probes), replace=False)
    for s, (po, pl) in zip(slots, probes):
        if 0 <= po and po + pl <= slab_len:
            o[s], ln[s] = po, pl
    o[0], ln[0] = lo, first_len
    o[-1], ln[-1] = hi - last_len, last_len
    return (ln.astype(np.uint64) << np.uint64(40)) | o.astype(np.uint64)


CASES = ["fits", "over_by_1", "unaligned_lo", "small", "slab_end", "reversed", "equal", "no_window", "wide"]


@pytest.mark.parametrize("shifts", [(0, 0), (8, 0), (0, 8)], ids=["aligned", "slab0_off8", "slab1_off8"])
@pytest.mark.parametrize("variant", sorted(STAGE_VARIANTS))
def test_staged_view_reads_the_slab_bytes_from_the_right_place(harness, variant, shifts):
    cols, cap = STAGE_VARIANTS[variant]
    rng = np.random.default_rng(variant * 10 + shifts[0] + 2 * shifts[1])
    slab_len = 4 * cap + 8192
    slabs = [rng.integers(0, 256, slab_len, dtype=np.uint8).tobytes() for _ in range(2)]
    nb = len(CASES)
    tail = 200  # the last block is partial: its window ends at row n - 1
    blocks = [[CASES[b], CASES[(b + 3) % nb]] for b in range(nb)]
    refs = np.zeros((nb * 256 - (256 - tail), 2), dtype=np.uint64)
    no_window = np.zeros((nb, 2), dtype=np.uint8)
    for b, pair in enumerate(blocks):
        r0, r1 = b * 256, min((b + 1) * 256, refs.shape[0])
        for c, case in enumerate(pair):
            refs[r0:r1, c] = block_refs(rng, case, cap, r1 - r0, slab_len)
            no_window[b, c] = case == "no_window"
    out, begin, flags = harness.staged(variant, refs, slabs, shifts, no_window)
    seen_shared = seen_slab = 0
    for c in range(cols):
        o, ln = refs[:, c] & np.uint64(OFF_MASK), refs[:, c] >> np.uint64(40)
        for b in range(nb):
            r0, r1 = b * 256, min((b + 1) * 256, refs.shape[0])
            want = staged_rule(o[r0:r1], ln[r0:r1], cap, not no_window[b, c], shifts[c] % 16 == 0)
            got = flags[r0:r1, c]
            assert np.array_equal(got, want.astype(np.uint8)), (c, blocks[b][c], int(np.flatnonzero(got != want)[0]))
            seen_shared += int(want.sum())
            seen_slab += int((~want).sum())
        for i in range(refs.shape[0]):
            b0, n = int(begin[2 * i + c]), int(ln[i])
            assert out[b0:b0 + n].tobytes() == slabs[c][int(o[i]):int(o[i]) + n], (c, i)
    if cols == 2 or shifts[0] == 0:
        assert seen_shared > 0 and seen_slab > 0
    assert (flags[:, cols:] == 0xFF).all()  # windows the functor does not have are never read


def test_staged_rule_cases_reach_both_sides_of_each_edge():
    """The block builder puts strings on both sides of the staged range's ends; at least one of each lands where the rule says."""
    rng = np.random.default_rng(3)
    cap, slab_len = 1024, 4 * 1024 + 8192
    for case in ("fits", "over_by_1", "unaligned_lo", "slab_end"):
        refs = block_refs(rng, case, cap, 256, slab_len)
        o, ln = refs & np.uint64(OFF_MASK), refs >> np.uint64(40)
        s = staged_rule(o, ln, cap, True, True)
        lo16 = int(o[0]) & ~15
        end = lo16 + min(((int(o[-1] + ln[-1]) - lo16 + 15) & ~15) + 16, cap)
        e = (o + ln).astype(np.int64)
        assert s[e == end - 16].any() and not s[e == end - 15].any(), case
        assert s[o.astype(np.int64) == lo16].any(), case
        if lo16:
            assert not s[o.astype(np.int64) == lo16 - 1].any(), case


# ------------------------------------------------------------------ the staged passes and the switches through the engine

FORMS = {"default": {}, "no_tma": {"GAR_NO_TMA": "1"}, "tma_all": {"GAR_TMA_ALL": "1"}}


def _subst(x, a, b):
    if isinstance(x, str):
        return x.replace(a, b)
    if isinstance(x, dict):
        return {k: _subst(v, a, b) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_subst(v, a, b) for v in x)
    return x


def long_string_model(seed, n_objects):
    """A randmodel cluster whose "kube-system" namespace is 300 bytes longer, consistently everywhere it appears (object keys,
    ingress load balancer names and so their hostnames, owner tags, TXT owner values).  Column-major, a block of 256 lbIngress
    hostnames then spans ~30 KB (over the tokeniser's 24 KB window) and a block of 256 records' values ~20 KB (over
    prepare_records' 16 KB value window)."""
    objects, actual = randmodel.make(seed, n_objects=n_objects)
    long_ns = "kube-system-" + "q" * 300
    return _subst(objects, "kube-system", long_ns), _subst(actual, "kube-system", long_ns)


def _windows_overflow(snap):
    """Some block of 256 rows has an lbIngress window over 24 KB, and some block of 256 records a value window over 16 KB."""
    ar = snap.arrays

    def widest(refs, begin=None, rows=None):
        spans = []
        for r0 in range(0, rows, 256):
            r1 = min(r0 + 256, rows)
            a, b = (r0, r1) if begin is None else (int(begin[r0]), int(begin[r1]))
            if b > a:
                spans.append(int(refs[b - 1] & OFF_MASK) + int(refs[b - 1] >> 40) - int(refs[a] & OFF_MASK))
        return max(spans)
    hn = ar["lbi_hostname"].astype(np.uint64)
    vals = ar["val_value"].astype(np.uint64)
    return widest(hn, rows=len(hn)) > 24 * 1024 and widest(vals, ar["rec_val_begin"], len(ar["rec_name"])) > 16 * 1024


def engine_in_form(garecon, monkeypatch, form, **kw):
    """An engine created with the form's switch set (the engine reads GAR_NO_TMA / GAR_TMA_ALL when it is created)."""
    for k in ("GAR_NO_TMA", "GAR_TMA_ALL"):
        monkeypatch.delenv(k, raising=False)
    for k, v in FORMS[form].items():
        monkeypatch.setenv(k, v)
    return garecon.Engine(**kw)


@pytest.mark.parametrize("seed", [1, 2])
def test_staged_windows_overflow_in_every_form(garecon, oracle, monkeypatch, seed):
    objects, actual = long_string_model(seed, 1500)
    snap = garecon.pack(objects, actual, layout="level")
    assert _windows_overflow(snap)
    want = oracle.diff(snap, "default", mode=1)
    results = {}
    for form in FORMS:
        with engine_in_form(garecon, monkeypatch, form, cluster_name="default") as e:
            e.load(snap)
            results[form], modes = [], []
            for _ in range(4):  # eager, eager on the prepared snapshot, recorded, replayed
                results[form].append(e.diff())
                modes.append(e.counters()["launch_mode"])
        assert modes == [0, 0, 1, 2], form
        for k, got in enumerate(results[form]):
            assert got.diff(want) == [], (form, k, got.describe_first_mismatch(want))
    for form in FORMS:
        for got in results[form]:
            assert got.diff(results["default"][0]) == []
