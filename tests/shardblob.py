"""The sharded exchange's blob layout (csrc/gar_shard.h) restated in numpy, for tests that check packed bytes.

A blob is one (source, destination) message: the levels of ShLevel one after the other, each laid out by `level_layout`: its
string-ref columns, u8 columns, u32 columns, global ids and child counts, every column starting 16-byte aligned, then its string
slab.  Inside a level's slab the strings follow row by row, column by column, each starting 8-byte aligned (`pad8`).  Bytes of a
string past its length up to the next 8-byte boundary, the alignment gaps and everything behind the last level are don't-care:
no reader may depend on them.

`expect_level` gives the exact bytes one packed level must hold; `live_mask` / `live_bytes` pick the bytes of a received blob
that carry data, so blobs of different exchange paths can be compared byte for byte."""
from __future__ import annotations

import numpy as np

L_OBJ, L_ANN, L_LBI, L_PORT, L_ACC, L_TAG, L_LIS, L_PR, L_EG, L_EP, L_REC, L_VAL, L_ZONE, L_LB, L_STUB, L_STUBTAG, L_PROBE = range(17)
L_NLEVELS = 17
LEVEL_NAMES = ["obj", "ann", "lbi", "port", "acc", "tag", "lis", "pr", "eg", "ep", "rec", "val", "zone", "lb", "stub", "stubtag", "probe"]
# (n_str, n_u8, n_u32, has_gid, n_child) per level: SH_SCHEMA
SCHEMA = [
    (2, 3, 1, 1, 3), (2, 0, 0, 0, 0), (1, 0, 0, 0, 0), (1, 0, 1, 0, 0), (2, 1, 0, 1, 2), (2, 0, 0, 0, 0), (0, 1, 0, 1, 2), (0, 0, 1, 0, 0),
    (0, 0, 0, 1, 1), (1, 0, 0, 0, 0), (2, 2, 1, 1, 1), (1, 0, 0, 1, 0), (1, 0, 0, 0, 0), (4, 1, 0, 1, 0), (2, 1, 0, 1, 1), (2, 0, 0, 0, 0),
    (1, 0, 1, 0, 0),
]
OFF_BITS = 40
OFF_MASK = (1 << OFF_BITS) - 1


def sh_align(x: int) -> int:
    return (x + 15) & ~15


def pad8(n):
    return (n + 7) & ~7


def gar_str(off, length):
    return (np.asarray(length, dtype=np.uint64) << np.uint64(OFF_BITS)) | np.asarray(off, dtype=np.uint64)


def level_layout(lvl: int, base: int, n: int, slab_bytes: int) -> dict:
    n_str, n_u8, n_u32, has_gid, n_child = SCHEMA[lvl]
    p = base
    L = {"str": [], "u8": [], "u32": [], "gid": None, "cnt": []}
    for _ in range(n_str):
        L["str"].append(p)
        p = sh_align(p + 8 * n)
    for _ in range(n_u8):
        L["u8"].append(p)
        p = sh_align(p + n)
    for _ in range(n_u32):
        L["u32"].append(p)
        p = sh_align(p + 4 * n)
    if has_gid:
        L["gid"] = p
        p = sh_align(p + 4 * n)
    for _ in range(n_child):
        L["cnt"].append(p)
        p = sh_align(p + 4 * n)
    L["slab"] = p
    L["end"] = sh_align(p + slab_bytes)
    return L


def level_layouts(meta_row) -> list[dict]:
    """Layouts of every level of one blob, from its meta row (rows per level, then slab bytes per level)."""
    out, p = [], 0
    for lvl in range(L_NLEVELS):
        L = level_layout(lvl, p, int(meta_row[lvl]), int(meta_row[L_NLEVELS + lvl]))
        out.append(L)
        p = L["end"]
    return out


def blob_bytes(meta_row) -> int:
    return level_layouts(meta_row)[-1]["end"]


def _spans(starts, lens):
    """Concatenated index ranges [starts[i], starts[i] + lens[i])."""
    starts = np.asarray(starts, dtype=np.int64).ravel()
    lens = np.asarray(lens, dtype=np.int64).ravel()
    total = int(lens.sum())
    if not total:
        return np.zeros(0, dtype=np.int64)
    first = np.cumsum(lens) - lens
    return np.repeat(starts - first, lens) + np.arange(total, dtype=np.int64)


def expect_level(lvl, base, rows, str_refs, u8c, u32c, gids, counts, slab, gap=None):
    """Exact bytes of one packed level of one destination.  rows = source rows in destination order; str_refs [n_str][n_src]
    uint64 refs into `slab` (uint8); u8c / u32c [k][n_src]; gids [n_src] (global id per source row) or None; counts
    [n_child][n_src] child counts per source row.  -> (layout, want bytes [L.end - base], care mask) relative to `base`.
    gap = None: the alignment gaps are don't-care; a byte value: they must still hold it (a buffer prefilled with it)."""
    n_str, n_u8, n_u32, has_gid, n_child = SCHEMA[lvl]
    rows = np.asarray(rows, dtype=np.int64)
    n = len(rows)
    refs = np.stack([np.asarray(str_refs[c], dtype=np.uint64)[rows] for c in range(n_str)], axis=1) if n_str else np.zeros((n, 0), np.uint64)
    lens = (refs >> np.uint64(OFF_BITS)).astype(np.int64)
    soff = (refs & np.uint64(OFF_MASK)).astype(np.int64)
    padded = pad8(lens)
    doff = (np.cumsum(padded.ravel()) - padded.ravel()).reshape(padded.shape) if padded.size else padded
    slab_bytes = int(padded.sum())
    L = level_layout(lvl, base, n, slab_bytes)
    size = L["end"] - base
    want = np.zeros(size, dtype=np.uint8)
    care = np.zeros(size, dtype=bool)

    def put(at, arr):
        b = np.ascontiguousarray(arr).view(np.uint8)
        want[at - base:at - base + len(b)] = b
        care[at - base:at - base + len(b)] = True

    for c in range(n_str):
        put(L["str"][c], gar_str(doff[:, c], lens[:, c]))
    for c in range(n_u8):
        put(L["u8"][c], np.asarray(u8c[c], dtype=np.uint8)[rows])
    for c in range(n_u32):
        put(L["u32"][c], np.asarray(u32c[c], dtype=np.uint32)[rows])
    if has_gid:
        put(L["gid"], np.asarray(gids, dtype=np.uint32)[rows])
    for c in range(n_child):
        put(L["cnt"][c], np.asarray(counts[c], dtype=np.uint32)[rows])
    s0 = L["slab"] - base
    care[s0:s0 + slab_bytes] = True
    want[_spans(s0 + doff, lens)] = np.asarray(slab, dtype=np.uint8)[_spans(soff, lens)]
    if gap is not None:
        want[~care] = gap
        care[:] = True
    # [len, pad8(len)) of every string: don't-care
    care[_spans(s0 + doff + lens, padded - lens)] = False
    return L, want, care


def parse_blob(blob, meta_row):
    """Columns of every level of one received blob: a list of dicts {str: [refs], u8: [..], u32: [..], gid, cnt: [..]}, plus
    structural checks: every string-ref column's offsets follow the row-major pad8 scan of the lengths and the level's strings
    fill exactly the slab bytes its meta row announces."""
    blob = np.asarray(blob, dtype=np.uint8)
    out = []
    for lvl, L in enumerate(level_layouts(meta_row)):
        n = int(meta_row[lvl])
        n_str, n_u8, n_u32, has_gid, n_child = SCHEMA[lvl]
        assert L["end"] <= len(blob), f"level {LEVEL_NAMES[lvl]} ends at {L['end']} past the blob ({len(blob)} bytes)"
        col = lambda at, dt, k: blob[at:at + k * np.dtype(dt).itemsize].view(dt)
        d = {"str": [col(a, np.uint64, n) for a in L["str"]], "u8": [col(a, np.uint8, n) for a in L["u8"]],
             "u32": [col(a, np.uint32, n) for a in L["u32"]], "gid": col(L["gid"], np.uint32, n) if has_gid else None,
             "cnt": [col(a, np.uint32, n) for a in L["cnt"]], "layout": L}
        if n_str and n:
            refs = np.stack(d["str"], axis=1)
            lens = (refs >> np.uint64(OFF_BITS)).astype(np.int64).ravel()
            offs = (refs & np.uint64(OFF_MASK)).astype(np.int64).ravel()
            want = np.cumsum(pad8(lens)) - pad8(lens)
            assert np.array_equal(offs, want), f"level {LEVEL_NAMES[lvl]}: string offsets are not the pad8 scan of the lengths"
            assert int(pad8(lens).sum()) == int(meta_row[L_NLEVELS + lvl]), f"level {LEVEL_NAMES[lvl]}: strings do not fill the slab"
        out.append(d)
    return out


def live_mask(blob, meta_row):
    """Bytes of a blob that carry data: every column's n elements and every string's [off, off + len)."""
    blob = np.asarray(blob, dtype=np.uint8)
    mask = np.zeros(len(blob), dtype=bool)
    for lvl, d in enumerate(parse_blob(blob, meta_row)):
        L, n = d["layout"], int(meta_row[lvl])
        for a in L["str"]:
            mask[a:a + 8 * n] = True
        for a in L["u8"]:
            mask[a:a + n] = True
        for a in L["u32"] + L["cnt"] + ([L["gid"]] if L["gid"] is not None else []):
            mask[a:a + 4 * n] = True
        if d["str"] and n:
            refs = np.concatenate(d["str"])
            mask[_spans(L["slab"] + (refs & np.uint64(OFF_MASK)).astype(np.int64), (refs >> np.uint64(OFF_BITS)).astype(np.int64))] = True
    return mask


def live_bytes(blob, meta_row):
    blob = np.asarray(blob, dtype=np.uint8)
    return blob[live_mask(blob, meta_row)]
