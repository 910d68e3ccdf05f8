"""GPU tier: the export's window-range copy and its pipelined gather-to-host (csrc/gar_engine.cu), against exact numpy references.

tests/cuda/export_harness.cu calls the engine's members on host arrays:
  * compact_copy(w0, w1)  k_compact_copy / k_compact_long over windows [w0, w1) only, into a buffer that starts at window w0:
                          ranges that start and end mid-string and mid-long-string, the last window, a range past the end
  * export_slab           the whole slab gathered EXPORT_CHUNK windows at a time through the ring of EXPORT_RING slots into a
                          host array: many chunks (the ring wraps), long strings over chunk boundaries, pageable and pinned
Every comparison is integer and bit-exact."""
import ctypes as C

import numpy as np
import pytest

from test_compact_kernels import GUARD, Harness, slab_of

pytestmark = pytest.mark.gpu

_u8p, _u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)


class ExportHarness(Harness):
    def __init__(self, path):
        super().__init__(path)
        lib = self.lib
        lib.ch_export_chunk.restype = C.c_uint32
        lib.ch_export_ring.restype = C.c_uint32
        lib.ch_compact_copy_range.argtypes = [C.c_void_p, _u64p, _u64p, C.c_uint32, _u8p, C.c_uint64, C.c_int, C.c_uint32, C.c_uint32, _u8p, C.c_uint64, C.c_uint32]
        lib.ch_export_slab.argtypes = [C.c_void_p, _u64p, _u64p, C.c_uint32, _u8p, C.c_uint64, C.c_int, _u8p]
        self.chunk, self.ring = int(lib.ch_export_chunk()), int(lib.ch_export_ring())

    @staticmethod
    def refs(slab, src_off, lens):
        src_off, lens = np.asarray(src_off, dtype=np.uint64), np.asarray(lens, dtype=np.uint64)
        sref = np.ascontiguousarray(src_off | (lens << np.uint64(40)))
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        total = int(off[-1])
        idx = np.repeat(src_off.astype(np.int64) - off[:-1].astype(np.int64), lens.astype(np.int64)) + np.arange(total, dtype=np.int64)
        return sref, off, total, np.ascontiguousarray(slab, dtype=np.uint8)[idx]

    def check_range(self, slab, src_off, lens, w0, w1):
        slab = np.ascontiguousarray(slab, dtype=np.uint8)
        sref, off, total, want = self.refs(slab, src_off, lens)
        lo, hi = min(w0 * self.window, total), min(w1 * self.window, total)
        out = np.zeros(hi - lo + GUARD, dtype=np.uint8)
        rc = self.lib.ch_compact_copy_range(self.h, sref.ctypes.data_as(_u64p), off.ctypes.data_as(_u64p), len(sref), slab.ctypes.data_as(_u8p), len(slab),
                                            int(bool((np.asarray(lens) > self.long).any())), w0, w1, out.ctypes.data_as(_u8p), hi - lo, GUARD)
        assert rc == 0, self.lib.ch_error(self.h).decode()
        assert np.array_equal(out[:hi - lo], want[lo:hi])
        assert (out[hi - lo:] == 0xCD).all()

    def check_export(self, slab, src_off, lens, out=None):
        slab = np.ascontiguousarray(slab, dtype=np.uint8)
        sref, off, total, want = self.refs(slab, src_off, lens)
        if out is None:
            out = np.empty(total + GUARD, dtype=np.uint8)
        out[:] = 0xCD
        rc = self.lib.ch_export_slab(self.h, sref.ctypes.data_as(_u64p), off.ctypes.data_as(_u64p), len(sref), slab.ctypes.data_as(_u8p), len(slab),
                                     int(bool((np.asarray(lens) > self.long).any())), out.ctypes.data_as(_u8p))
        assert rc == 0, self.lib.ch_error(self.h).decode()
        assert np.array_equal(out[:total], want)
        assert (out[total:] == 0xCD).all()
        return total


@pytest.fixture(scope="module")
def hx():
    import __graft_entry__ as ge
    h = ExportHarness(ge.build_backend_harness(name="export_harness"))
    yield h
    h.close()


def test_range_of_short_strings_starts_and_ends_mid_string(hx):
    rng = np.random.default_rng(3)
    lens = rng.integers(20, 81, size=20_000)
    slab = slab_of(int(lens.sum()) + 100, 4)
    src = (np.concatenate([[0], np.cumsum(lens)[:-1]]) + 5)[rng.permutation(len(lens))]
    windows = -(-int(lens.sum()) // hx.window)
    for w0, w1 in ((0, 1), (1, 2), (3, 7), (windows - 2, windows), (windows - 1, windows + 5), (0, windows)):
        hx.check_range(slab, src, lens, w0, w1)


def test_range_starts_and_ends_inside_long_strings(hx):
    w, L = hx.window, hx.long
    slab = slab_of(8 * w, 5)
    lens = [300, 3 * w + 77, L + 1, 40, 2 * w - 13, 9]  # a range boundary falls inside each long string
    src = [1, 7, 3 * w + 200, 50, 4 * w + 3, 11]
    total = sum(lens)
    for w0 in range(0, -(-total // w)):
        for w1 in (w0 + 1, w0 + 2, w0 + 3):
            hx.check_range(slab, src, lens, w0, w1)


def test_whole_range_as_chunks_equals_numpy(hx):
    """Windows run chunk by chunk through the ring: more chunks than ring slots, so every slot is reused several times."""
    rng = np.random.default_rng(9)
    lens = rng.integers(0, 400, size=400_000)
    lens[::997] = rng.integers(hx.long + 1, 3 * hx.window, size=len(lens[::997]))
    slab = slab_of(int(lens.max()) + 200_000, 10)
    src = rng.integers(0, 200_000, size=len(lens))
    total = hx.check_export(slab, src, lens)
    assert total > 2 * hx.ring * hx.chunk * hx.window


def test_long_string_over_chunk_boundaries(hx):
    chunk_bytes = hx.chunk * hx.window
    slab = slab_of(2 * chunk_bytes + 4096, 12)
    for lead in (0, 1, 15, 16, chunk_bytes - 3):
        hx.check_export(slab, [0, 3, 9], [lead, 2 * chunk_bytes + 1000, 5])


def test_empty_and_tiny(hx):
    slab = slab_of(1000, 13)
    assert hx.check_export(slab, np.arange(100), np.zeros(100, dtype=np.int64)) == 0
    hx.check_export(slab, [5], [1])


def test_pinned_destination(hx):
    import torch
    rng = np.random.default_rng(14)
    lens = rng.integers(1, 300, size=150_000)
    slab = slab_of(100_000, 15)
    src = rng.integers(0, 99_000, size=len(lens))
    out = torch.empty(int(lens.sum()) + GUARD, dtype=torch.uint8, pin_memory=True).numpy()
    hx.check_export(slab, src, lens, out)
