"""GPU tier: the sharded exchange's data-path kernels (csrc/gar_shard.h, gar_engine.cu), one at a time, against the blob layout
restated in numpy (tests/shardblob.py).

tests/cuda/shard_pack_harness.cu packs ONE level of a synthetic source into G destinations with the engine's own plan and
Sharder::pack_to, either with the default pack (k_for_each<FShPackRows>, strings cut at SH_LONG_WORDS, FShPackLong finishes them)
or with the bulk-store pack (k_shard_pack_rows: a block's slab range assembled in shared memory and written by one bulk store with
8-byte head and tail stores; blocks that straddle two destinations, exceed PACK_TILE or carry no string bytes store per thread).
The destination buffer starts as a sentinel byte.  For every destination: every column byte and every string byte must be exact,
and every byte that is neither (alignment gaps, bytes behind the level, guard bands) must still be the sentinel.  The only
don't-care bytes are those of a string past its length up to the next 8-byte boundary.

k_peer_push is checked the same way on 1..7 descriptors of different lengths around its grid stride.

The shapes are built on the host so that the bulk-store pack's `s_staged` rule is met and missed for the reasons it has
(test_pack_cases_reach_both_sides_of_the_staged_rule runs without a GPU)."""
import ctypes as C

import numpy as np
import pytest

import shardblob as sb

_u8p, _u32p, _u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)

PACK_TILE = 40 * 1024
SH_LONG_WORDS = 256
SH_LONG_STRIDE = 132 * 8 * 256 // 8  # rows between two visits of one FShPackLong worker
PUSH_STRIDE = 24 * 512               # uint4 per grid stride of k_peer_push
SENTINEL, PAD_BYTE = 0xA5, 0x5A
GUARD = 64


class Harness:
    def __init__(self, path):
        lib = self.lib = C.CDLL(str(path))
        lib.sph_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        lib.sph_destroy.argtypes = [C.c_void_p]
        lib.sph_error.argtypes = [C.c_void_p]
        lib.sph_error.restype = C.c_char_p
        lib.sph_constants.argtypes = [_u64p]
        lib.sph_pack.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint32, _u8p, C.c_uint64, C.c_uint8, _u64p, _u8p, _u32p, _u32p, C.c_uint32, _u32p,
                                 C.c_uint32, _u32p, C.c_uint32, _u32p, _u64p, C.c_uint8, C.c_uint64, _u8p, _u32p]
        lib.sph_push.argtypes = [C.c_void_p, C.c_int, _u64p, _u8p, C.c_uint64, C.c_uint8, _u8p]
        self.h = C.c_void_p()
        assert lib.sph_create(0, C.byref(self.h)) == 0, lib.sph_error(None).decode()

    def _ok(self, rc):
        assert rc == 0, self.lib.sph_error(self.h).decode()

    def constants(self):
        out = np.zeros(7, dtype=np.uint64)
        self.lib.sph_constants(out.ctypes.data_as(_u64p))
        return [int(x) for x in out]

    def pack(self, c, tma):
        n_str, n_u8, n_u32, has_gid, n_child = sb.SCHEMA[c.lvl]
        a = lambda x, dt: np.ascontiguousarray(x if x is not None and len(x) else np.zeros(1), dtype=dt)
        slab, strs, u8c, u32c = a(c.slab, np.uint8), a(np.concatenate(c.strs) if n_str else None, np.uint64), a(
            np.concatenate(c.u8c) if n_u8 else None, np.uint8), a(np.concatenate(c.u32c) if n_u32 else None, np.uint32)
        gid = a(c.gid, np.uint32) if c.gid is not None else None
        cb = a(np.concatenate(c.child_begin) if n_child else None, np.uint32)
        sel, row_off, dst = a(c.sel, np.uint32), a(c.row_off, np.uint32), a(c.dst_off, np.uint64)
        out = np.zeros(c.out_len, dtype=np.uint8)
        scan = np.zeros(len(c.sel) + 1, dtype=np.uint32)
        self._ok(self.lib.sph_pack(self.h, c.lvl, int(tma), c.G, slab.ctypes.data_as(_u8p), len(c.slab), PAD_BYTE, strs.ctypes.data_as(_u64p),
                                   u8c.ctypes.data_as(_u8p), u32c.ctypes.data_as(_u32p), gid.ctypes.data_as(_u32p) if gid is not None else None,
                                   c.gid_base, cb.ctypes.data_as(_u32p), c.n, sel.ctypes.data_as(_u32p), len(c.sel), row_off.ctypes.data_as(_u32p),
                                   dst.ctypes.data_as(_u64p), SENTINEL, c.out_len, out.ctypes.data_as(_u8p), scan.ctypes.data_as(_u32p)))
        return out, scan

    def push(self, n16, src):
        n16 = np.ascontiguousarray(n16, dtype=np.uint64)
        out = np.zeros(int(16 * n16.sum()) + 2 * GUARD * len(n16), dtype=np.uint8)
        src = np.ascontiguousarray(src, dtype=np.uint8)
        self._ok(self.lib.sph_push(self.h, len(n16), n16.ctypes.data_as(_u64p), src.ctypes.data_as(_u8p), GUARD, SENTINEL, out.ctypes.data_as(_u8p)))
        return out

    def close(self):
        if self.h:
            self.lib.sph_destroy(self.h)
            self.h = C.c_void_p()


@pytest.fixture(scope="module")
def harness():
    import __graft_entry__ as ge
    h = Harness(ge.build_backend_harness(name="shard_pack_harness"))
    yield h
    h.close()


# ------------------------------------------------------------------ synthetic levels

class Case:
    """One level of one source rank: source columns, a selection grouped by destination, and where each destination's level
    starts in the output buffer (16-aligned, with guard bands between the destinations)."""

    def __init__(self, name, lvl, lens, dest_rows, seed, phases=None, gid_explicit=False, slab_end_row=None):
        rng = np.random.default_rng(seed)
        n_str, n_u8, n_u32, has_gid, n_child = sb.SCHEMA[lvl]
        lens = np.asarray(lens, dtype=np.int64).reshape(-1, n_str) if n_str else np.zeros((len(lens), 0), np.int64)
        self.name, self.lvl, self.G, self.n = name, lvl, len(dest_rows), len(lens)
        # the source slab: strings in row order at varied 8-byte phases (or the given ones), random bytes everywhere else
        offs = np.zeros(lens.shape, dtype=np.int64)
        p = 0
        for i, r in enumerate(lens):
            for c, ln in enumerate(r):
                want = int(phases[i, c]) if phases is not None else int(rng.integers(0, 8))
                p += (want - p) % 8 + 8 * int(rng.integers(0, 2))
                offs[i, c] = p
                p += int(ln)
        self.slab = rng.integers(0, 256, p, dtype=np.uint8)
        if slab_end_row is not None:  # the last string of this row ends on the slab's last byte
            r, c = slab_end_row
            assert offs[r, c] + lens[r, c] == p
        self.strs = [sb.gar_str(offs[:, c], lens[:, c]) for c in range(n_str)]
        self.u8c = [rng.integers(0, 256, self.n, dtype=np.uint8) for _ in range(n_u8)]
        self.u32c = [rng.integers(0, 2 ** 32, self.n, dtype=np.uint64).astype(np.uint32) for _ in range(n_u32)]
        self.gid_base = int(rng.integers(0, 1 << 20))
        self.gid = rng.permutation(self.n).astype(np.uint32) * 3 + 7 if gid_explicit else None
        self.counts = [rng.integers(0, 4, self.n).astype(np.uint32) for _ in range(n_child)]
        self.child_begin = [np.concatenate([[0], np.cumsum(k)]).astype(np.uint32) for k in self.counts]
        self.sel = np.concatenate([np.asarray(r, dtype=np.uint32) for r in dest_rows]) if dest_rows else np.zeros(0, np.uint32)
        self.row_off = np.concatenate([[0], np.cumsum([len(r) for r in dest_rows])]).astype(np.uint32)
        self.dest_rows = [np.asarray(r, dtype=np.int64) for r in dest_rows]
        # host restatement of the plan's slab scan and of every destination's layout
        row_bytes = sb.pad8(lens).sum(axis=1) if n_str else np.zeros(self.n, np.int64)
        self.scan = np.concatenate([[0], np.cumsum(row_bytes[self.sel.astype(np.int64)])]).astype(np.int64)
        self.dst_off, p = [], GUARD
        for d in range(self.G):
            self.dst_off.append(p)
            L = sb.level_layout(lvl, p, len(dest_rows[d]), int(self.scan[self.row_off[d + 1]] - self.scan[self.row_off[d]]))
            p = L["end"] + GUARD
        self.out_len = p + GUARD

    def gids(self):
        return self.gid if self.gid is not None else (self.gid_base + np.arange(self.n)).astype(np.uint32)

    def expect(self):
        """(want, care) over the whole output buffer: sentinel everywhere outside the packed bytes."""
        want = np.full(self.out_len, SENTINEL, dtype=np.uint8)
        care = np.ones(self.out_len, dtype=bool)
        for d in range(self.G):
            L, w, c = sb.expect_level(self.lvl, self.dst_off[d], self.dest_rows[d], self.strs, self.u8c, self.u32c, self.gids(), self.counts, self.slab,
                                      gap=SENTINEL)
            want[self.dst_off[d]:L["end"]] = w
            care[self.dst_off[d]:L["end"]] = c
        return want, care

    def dest_of(self, j):
        d = 0
        while d + 1 < self.G and j >= self.row_off[d + 1]:
            d += 1
        return d

    def blocks(self):
        """k_shard_pack_rows' s_staged rule per block, restated: -> list of (staged, reason, head, body, tail)."""
        n_str = sb.SCHEMA[self.lvl][0]
        m, out = len(self.sel), []
        for j0 in range(0, m, 256):
            j1 = min(j0 + 256, m)
            d0, d1 = self.dest_of(j0), self.dest_of(j1 - 1)
            lo, hi = int(self.scan[j0]), int(self.scan[j1])
            if not n_str:
                out.append((False, "no_strings", 0, 0, 0))
            elif d0 != d1:
                out.append((False, "straddles", 0, 0, 0))
            elif hi == lo:
                out.append((False, "empty", 0, 0, 0))
            elif hi - lo > PACK_TILE:
                out.append((False, "over_tile", 0, 0, 0))
            else:
                L = sb.level_layout(self.lvl, self.dst_off[d0], len(self.dest_rows[d0]), 0)
                dst = L["slab"] + lo - int(self.scan[self.row_off[d0]])
                head = min(8 if dst & 15 else 0, hi - lo)
                body = (hi - lo - head) & ~15
                out.append((True, "exact_tile" if hi - lo == PACK_TILE else "staged", head, body, hi - lo - head - body))
        return out

    def any_long(self):
        return any(int(sb.pad8((s[self.sel] >> np.uint64(40)).astype(np.int64)).max(initial=0)) > 8 * SH_LONG_WORDS for s in self.strs)


def spread(n, G, rng, empty=()):
    """n rows split over G destinations (the ones in `empty` get none), rows ascending inside each destination."""
    keep = [d for d in range(G) if d not in empty]
    cuts = np.sort(rng.choice(np.arange(1, n), size=len(keep) - 1, replace=False))  # every kept destination gets a row
    parts = np.split(rng.permutation(n), cuts)
    out, k = [], 0
    for d in range(G):
        if d in empty:
            out.append([])
        else:
            out.append(sorted(parts[k].tolist()))
            k += 1
    return out


def by_bounds(bounds):
    """Destination row lists for a selection of the identity rows 0..bounds[-1] cut at `bounds`."""
    return [list(range(bounds[d], bounds[d + 1])) for d in range(len(bounds) - 1)]


def block_bytes_case(name, lvl, sizes, seed):
    """One destination, 256 rows per block; block b's rows carry exactly sizes[b] slab bytes in one string (0: a block of empty
    strings), so each block's range and the destination phase of the next one are chosen."""
    n_str = sb.SCHEMA[lvl][0]
    lens = np.zeros((256 * len(sizes), n_str), dtype=np.int64)
    rng = np.random.default_rng(seed)
    for b, size in enumerate(sizes):
        if size:
            lens[256 * b + int(rng.integers(0, 256)), -1] = size - int(rng.integers(0, 8))  # pad8(len) == size
    return Case(name, lvl, lens, [list(range(len(lens)))], seed)


LENS = [0, 1, 7, 8, 9, 2040, 2047, 2048, 2049, 2056, 2057]


def cases():
    rng = np.random.default_rng(11)
    out = []
    # row counts around the block size, destinations with no rows, 1..8 destinations
    for m, G, empty in [(1, 1, ()), (255, 2, (0,)), (256, 3, (1,)), (257, 8, (0, 3, 7)), (511, 5, (4,)), (4097, 8, (2, 5))]:
        lens = rng.integers(0, 300, (m + 50, 2))
        out.append(Case(f"m{m}_G{G}", sb.L_ANN, lens, spread(m, G, rng, empty), seed=m))
    # destination boundaries at a block edge and one row either side of it: blocks straddle two destinations
    out.append(Case("bounds_256k", sb.L_ANN, rng.integers(0, 200, (1100, 2)), by_bounds([0, 0, 255, 512, 513, 767, 769, 1024, 1024]), seed=5))
    # block ranges of 8, 16, 24, 32 bytes at destination phases 0 and 8, empty blocks, exactly PACK_TILE and PACK_TILE + 8
    out.append(block_bytes_case("block_bytes", sb.L_ANN, [8, 8, 16, 16, 8, 24, 24, 8, 32, 0, 32, 16, 0, 24, 8, PACK_TILE, 8, PACK_TILE + 8, 16], seed=6))
    # string lengths around the 8-byte word and the 2 KB cut at every source phase; one string ends on the slab's last byte
    lens = np.array([[ln, ln2] for ln in LENS for ln2 in LENS], dtype=np.int64)
    phases = np.arange(lens.size).reshape(lens.shape) % 8
    dense = Case("lengths_dense", sb.L_ANN, lens, [list(range(len(lens)))], seed=7, phases=phases, slab_end_row=(len(lens) - 1, 1))
    out.append(dense)
    sparse = np.zeros((256 * len(lens), 2), dtype=np.int64)  # one such row per block: every block is staged (<= PACK_TILE)
    sparse[255::256] = lens
    ph = np.zeros(sparse.shape, dtype=np.int64)
    ph[255::256] = phases
    out.append(Case("lengths_per_block", sb.L_ANN, sparse, by_bounds([0, 256 * 40, 256 * 81, len(sparse)]), seed=8, phases=ph,
                    slab_end_row=(len(sparse) - 1, 1)))
    # a > 40 KB string among staged 2-40 KB ones: its block leaves the tile, the long pass runs and rewrites the staged strings too
    mixed = np.zeros((256 * 12, 2), dtype=np.int64)
    for b in range(12):
        mixed[256 * b + 3, 1] = int(rng.integers(2049, 20000))
        mixed[256 * b + 100, 0] = int(rng.integers(2049, 20000))
    mixed[256 * 7 + 50, 1] = 50_000
    out.append(Case("long_among_staged", sb.L_ANN, mixed, [list(range(len(mixed)))], seed=9))
    # more rows than one stride of FShPackLong's workers, long strings beyond it
    m = SH_LONG_STRIDE + 6000
    wrap = rng.integers(0, 40, (m, 2))
    wrap[rng.choice(np.arange(SH_LONG_STRIDE, m), 60, replace=False), 1] = rng.integers(2049, 9000, 60)
    wrap[rng.choice(SH_LONG_STRIDE, 20, replace=False), 0] = rng.integers(2049, 9000, 20)
    wrap[m - 1, 1] = 2057
    out.append(Case("long_pass_wraps", sb.L_ANN, wrap, by_bounds([0, 10_000, 20_001, m]), seed=10))
    # a source row selected for two destinations (record sets replicated to several homes, LevelPlan::multi)
    base = spread(900, 4, rng)
    dup = [sorted(set(r) | set(rng.choice(900, 120, replace=False).tolist())) for r in base]
    out.append(Case("multi", sb.L_ANN, rng.integers(0, 400, (900, 2)), dup, seed=12))
    # the other schemas: 4 strings + gid (LB, explicit gids as after round 1), 2 strings + u8/u32/gid/3 child links (OBJ),
    # no strings (LIS: the bulk-store pack always stores per thread, no long pass)
    out.append(Case("lb", sb.L_LB, rng.integers(0, 120, (1300, 4)), spread(1300, 3, rng, (1,)), seed=13, gid_explicit=True))
    obj = rng.integers(0, 90, (800, 2))
    obj[[5, 400, 799], 0] = [2049, 4100, 2056]
    out.append(Case("obj", sb.L_OBJ, obj, spread(800, 4, rng), seed=14))
    out.append(Case("lis", sb.L_LIS, np.zeros(1500), spread(1500, 5, rng, (2,)), seed=15))
    return out


CASES = cases()


def test_pack_cases_reach_both_sides_of_the_staged_rule():
    """Every reason k_shard_pack_rows has to store per thread occurs, staged blocks reach all four (head, tail) store shapes,
    with and without a bulk body, and ranges of exactly PACK_TILE; the long-string pass runs with and without a second stride."""
    blocks = [b for c in CASES for b in c.blocks()]
    reasons = {r: sum(1 for b in blocks if b[1] == r) for r in ("staged", "exact_tile", "straddles", "empty", "over_tile", "no_strings")}
    assert all(reasons.values()), reasons
    shapes = {(h, t, body > 0) for s, _, h, body, t in blocks if s}
    for h in (0, 8):
        for t in (0, 8):
            assert (h, t, True) in shapes, (h, t, shapes)
    assert {(0, 8, False), (8, 0, False), (8, 8, False)} <= shapes, shapes
    long_cases = [c for c in CASES if c.any_long()]
    assert any(len(c.sel) > SH_LONG_STRIDE for c in long_cases) and any(len(c.sel) <= SH_LONG_STRIDE for c in long_cases)
    wrap = next(c for c in CASES if c.name == "long_pass_wraps")
    assert (sb.pad8((wrap.strs[1][wrap.sel[SH_LONG_STRIDE:]] >> np.uint64(40)).astype(np.int64)) > 8 * SH_LONG_WORDS).sum() >= 50
    print("s_staged blocks:", reasons)


def _first_bad(got, want, care, case):
    bad = np.flatnonzero(care & (got != want))
    if not len(bad):
        return ""
    k = int(bad[0])
    where = "outside every destination's level"
    for d in range(case.G):
        L = sb.level_layout(case.lvl, case.dst_off[d], len(case.dest_rows[d]), int(case.scan[case.row_off[d + 1]] - case.scan[case.row_off[d]]))
        if case.dst_off[d] <= k < L["end"]:
            where = f"destination {d}, level byte {k - case.dst_off[d]} (slab at {L['slab'] - case.dst_off[d]}, end {L['end'] - case.dst_off[d]})"
    return f"{len(bad)} wrong bytes, first at {k}: {where}: got {got[k]:#x} want {want[k]:#x}"


@pytest.mark.gpu
def test_harness_constants_match_the_restatement(harness):
    tile, long_words, workers, lanes, push_stride, pad, nlev = harness.constants()
    assert (tile, long_words, workers // lanes, push_stride, nlev) == (PACK_TILE, SH_LONG_WORDS, SH_LONG_STRIDE, PUSH_STRIDE, sb.L_NLEVELS)
    assert pad == 32


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_pack_level_is_exact(harness, case):
    want, care = case.expect()
    got = {}
    for tma in (0, 1):
        out, scan = harness.pack(case, tma)
        assert np.array_equal(scan.astype(np.int64), case.scan), "the plan's slab scan"
        bad = _first_bad(out, want, care, case)
        assert not bad, f"{'bulk-store' if tma else 'default'} pack: {bad}"
        got[tma] = out
    assert np.array_equal(got[0][care], got[1][care])


# ------------------------------------------------------------------ k_peer_push

PUSH_SETS = [
    [0], [1], [PUSH_STRIDE - 1], [PUSH_STRIDE], [4 * PUSH_STRIDE - 1], [4 * PUSH_STRIDE], [4 * PUSH_STRIDE + 1],
    [1, PUSH_STRIDE, 4 * PUSH_STRIDE + 1],
    [0, 4 * PUSH_STRIDE - 1, 2_000_003, 1, PUSH_STRIDE - 1, 4 * PUSH_STRIDE, 3 * PUSH_STRIDE + 5],
    [1_000_000, 3_000_017],
]


@pytest.mark.gpu
@pytest.mark.parametrize("n16", PUSH_SETS, ids=["-".join(map(str, s)) for s in PUSH_SETS])
def test_peer_push_copies_every_uint4_and_nothing_else(harness, n16):
    rng = np.random.default_rng(sum(n16) + len(n16))
    src = rng.integers(0, 256, 16 * sum(n16), dtype=np.uint8)
    out = harness.push(n16, src)
    so, oo = 0, 0
    for k, n in enumerate(n16):
        b = 16 * n
        dst = out[oo:oo + b + 2 * GUARD]
        assert (dst[:GUARD] == SENTINEL).all() and (dst[GUARD + b:] == SENTINEL).all(), f"descriptor {k}: a guard band was written"
        bad = np.flatnonzero(dst[GUARD:GUARD + b] != src[so:so + b])
        assert not len(bad), f"descriptor {k} (n16 {n}): {len(bad)} wrong bytes, first at uint4 {int(bad[0]) // 16}"
        so += b
        oo += b + 2 * GUARD
