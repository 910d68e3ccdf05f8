"""GPU tier: the CUDA primitives of the slab compaction (csrc/gar_engine.cu), one at a time, against exact numpy references.

tests/cuda/compact_harness.cu calls the engine's members on host arrays:
  * exclusive_scan(u64)  the look-back scan instantiated for 64-bit elements: running sums beyond 2^32, every tile-count boundary
  * compact_copy         k_compact_copy (windows assembled in shared memory, one bulk store each, the last window's tail by
                         ordinary stores) and k_compact_long (strings longer than COMPACT_LONG, 16-byte copies with a head and a
                         tail, sources at every phase of a 16-byte line)
Every comparison is integer and bit-exact."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

_u8p, _u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)
SCAN_TILE = 2048  # 256 threads x 8 items; the look-back reads 32 predecessor tiles per step
GUARD = 64


class Harness:
    def __init__(self, path):
        lib = self.lib = C.CDLL(str(path))
        lib.ch_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        lib.ch_destroy.argtypes = [C.c_void_p]
        lib.ch_error.argtypes = [C.c_void_p]
        lib.ch_error.restype = C.c_char_p
        lib.ch_window.restype = C.c_uint32
        lib.ch_long.restype = C.c_uint32
        lib.ch_exclusive_scan64.argtypes = [C.c_void_p, _u64p, C.c_uint32]
        lib.ch_compact_copy.argtypes = [C.c_void_p, _u64p, _u64p, C.c_uint32, _u8p, C.c_uint64, C.c_int, _u8p, C.c_uint32]
        self.h = C.c_void_p()
        rc = lib.ch_create(0, C.byref(self.h))
        assert rc == 0, lib.ch_error(None).decode()
        self.window, self.long = int(lib.ch_window()), int(lib.ch_long())

    def scan64(self, x):
        d = np.ascontiguousarray(x, dtype=np.uint64).copy()
        rc = self.lib.ch_exclusive_scan64(self.h, d.ctypes.data_as(_u64p), len(d))
        assert rc == 0, self.lib.ch_error(self.h).decode()
        return d

    def copy(self, slab, src_off, lens, any_long=None):
        """Strings (src_off[p], lens[p]) of `slab` copied back to back.  -> (output with GUARD bytes behind it, expected bytes)."""
        src_off, lens = np.asarray(src_off, dtype=np.uint64), np.asarray(lens, dtype=np.uint64)
        sref = np.ascontiguousarray(src_off | (lens << np.uint64(40)))
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        total = int(off[-1])
        out = np.zeros(total + GUARD, dtype=np.uint8)
        slab = np.ascontiguousarray(slab, dtype=np.uint8)
        if any_long is None:
            any_long = bool((lens > self.long).any())
        backing = np.zeros(1, dtype=np.uint64)
        rc = self.lib.ch_compact_copy(self.h, (sref if len(sref) else backing).ctypes.data_as(_u64p), off.ctypes.data_as(_u64p), len(sref),
                                      slab.ctypes.data_as(_u8p), len(slab), int(any_long), out.ctypes.data_as(_u8p), GUARD)
        assert rc == 0, self.lib.ch_error(self.h).decode()
        ln = lens.astype(np.int64)
        idx = np.repeat(src_off.astype(np.int64) - off[:-1].astype(np.int64), ln) + np.arange(total, dtype=np.int64)
        return out, slab[idx]

    def check(self, slab, src_off, lens, any_long=None):
        out, want = self.copy(slab, src_off, lens, any_long)
        assert np.array_equal(out[:len(want)], want)
        assert (out[len(want):] == 0xCD).all()  # nothing behind the new slab_len is written

    def close(self):
        self.lib.ch_destroy(self.h)


@pytest.fixture(scope="module")
def hz():
    import __graft_entry__ as ge
    h = Harness(ge.build_backend_harness(name="compact_harness"))
    yield h
    h.close()


def slab_of(n, seed):
    return np.random.default_rng(seed).integers(1, 255, size=n, dtype=np.uint8)


# ------------------------------------------------------------------ the 64-bit scan

@pytest.mark.parametrize("n", [1, 7, 8, 9, SCAN_TILE - 1, SCAN_TILE, SCAN_TILE + 1, 2 * SCAN_TILE, 31 * SCAN_TILE, 32 * SCAN_TILE, 32 * SCAN_TILE + 1,
                               33 * SCAN_TILE, 33 * SCAN_TILE + 5, 64 * SCAN_TILE, 65 * SCAN_TILE - 3, 200 * SCAN_TILE + 77])
def test_scan64_crosses_2_pow_32_at_every_tile_boundary(hz, n):
    """Lengths only (no bytes are allocated for them): values up to the legal 16 MiB string maximum, so the running sum passes
    2^32 inside the first few hundred elements; tile counts on both sides of one tile, of one look-back step (32 tiles) and of two."""
    x = np.random.default_rng(n).integers(0, 1 << 24, size=n, dtype=np.uint64)
    if n >= 300:
        x[:300] = (1 << 24) - 1  # 300 strings of the maximum length already exceed 2^32
    want = np.concatenate([[0], np.cumsum(x)[:-1]]).astype(np.uint64)
    got = hz.scan64(x)
    assert np.array_equal(got, want)
    if n >= 300:
        assert int(got[-1]) > 1 << 32


def test_scan64_of_zeros_and_ones(hz):
    assert not hz.scan64(np.zeros(5 * SCAN_TILE + 3, dtype=np.uint64)).any()
    n = 40 * SCAN_TILE + 11
    assert np.array_equal(hz.scan64(np.ones(n, dtype=np.uint64)), np.arange(n, dtype=np.uint64))


# ------------------------------------------------------------------ the window copy

def test_copy_short_strings_across_many_windows(hz):
    """20-80 byte strings gathered from shuffled sources: windows start and end mid-string, sources sit at every alignment."""
    rng = np.random.default_rng(1)
    lens = rng.integers(20, 81, size=20_000)
    slab = slab_of(int(lens.sum()) + 100, 2)
    order = rng.permutation(len(lens))
    src = np.zeros(len(lens), dtype=np.int64)
    src[order] = np.concatenate([[0], np.cumsum(lens[order])[:-1]]) + 3
    assert set((src % 16).tolist()) == set(range(16))
    hz.check(slab, src, lens)


@pytest.mark.parametrize("align", range(16))
def test_copy_source_alignment(hz, align):
    """Every source phase against destination phases 0..15 (a leading string of k bytes shifts the rest), short and long strings."""
    slab = slab_of(3 * hz.window + 6000, 3 + align)
    for lead in range(16):
        lens = [lead, 5, hz.long, hz.long + 1, 40, hz.long + 17 + lead, 2 * hz.window + 33, 9]
        src = [0, 16 + align, 64 + align, 2000 + align, 4000 + align, 4100 + align, 5500 + align, 100 + align]
        hz.check(slab, src, lens)


def test_copy_strings_straddling_two_and_three_windows(hz):
    w = hz.window
    slab = slab_of(4 * w, 5)
    # below the long-string threshold a string straddles at most two windows: place 1000-byte strings over every window boundary
    lens = [w - 500, 1000, w - 1000, 1000, 7]
    hz.check(slab, [0, 11, 1011, 77, 3], lens)
    # a long string that begins in window 0, covers window 1 completely and ends in window 2 (three windows), and one that covers
    # windows exactly (nothing to assemble in them)
    hz.check(slab, [5, 100, 9], [100, 2 * w + 50, 30])
    hz.check(slab, [0, 33, 1], [w, 2 * w, 16])


def test_copy_windows_of_empty_strings(hz):
    w = hz.window
    slab = slab_of(3 * w, 6)
    lens = np.zeros(5000, dtype=np.int64)
    hz.check(slab, np.arange(5000) % 97, lens)  # total == 0: no launch at all
    lens = np.concatenate([[w], np.zeros(3000, dtype=np.int64), [w], np.zeros(3000, dtype=np.int64), [12]])  # empties exactly on window boundaries
    hz.check(slab, np.arange(len(lens)) % 50, lens)
    lens = np.concatenate([[40], np.zeros(100_000, dtype=np.int64), [40]])  # a long run of empties inside one window
    hz.check(slab, np.arange(len(lens)) % 50, lens)


@pytest.mark.parametrize("tail", [0, 1, 15, 16, 17, 31])
def test_copy_last_window(hz, tail):
    """The last window is shorter than the others: its multiple of 16 bytes goes out by the bulk store, the rest by ordinary stores."""
    w = hz.window
    slab = slab_of(2 * w, 7)
    for total in (tail, w + tail, 2 * w - 16 + tail):
        if total == 0:
            continue
        lens = np.full(total // 30, 30, dtype=np.int64)
        lens = np.concatenate([lens, [total - int(lens.sum())]])
        hz.check(slab, np.arange(len(lens)) * 7 % 1000, lens)


def test_copy_long_threshold_head_and_tail(hz):
    """Lengths around COMPACT_LONG; long strings whose destination starts at every phase (head of 0..15 bytes) and whose length
    leaves every tail (0..15 bytes)."""
    L = hz.long
    slab = slab_of(8 * L + 4096, 8)
    for lead in range(16):
        for extra in range(16):
            hz.check(slab, [0, 7, 1 + extra], [lead, L + 1 + extra, 3])
    hz.check(slab, [0, 5, 9, 13, 17], [L - 1, L, L + 1, L + 2, 2 * L])
    out, want = hz.copy(slab, [0, 5, 9], [L - 1, L, 10], any_long=True)  # the long launch with nothing to do
    assert np.array_equal(out[:len(want)], want)
