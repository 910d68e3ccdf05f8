"""Object deltas at table level: the rules of gar_snapshot_apply_objects (include/garecon.h) on numpy column dicts, and a
seeded churn generator of informer-like batches.

ColumnMirror holds the object table a full gar_snapshot_load would need after a sequence of deltas, laid out like the
engine's resident table: its slab is the loaded slab followed by every delta's upsert slab at a 16-byte aligned offset,
so the mirror's string references (and therefore tok_name / tok_region of a diff) are bit-identical to the engine's.
profiles/delta_bench.py and the GPU tests use both; the CPU tests use a dict-level mirror (tests/test_object_deltas.py).
"""
from __future__ import annotations

import numpy as np

from . import tables

GAR_NONE = 0xFFFFFFFF
_MASK = np.uint64((1 << 40) - 1)
ANN_R53 = b"aws-global-accelerator-controller.h3poteto.dev/route53-hostname"
ANN_LISTEN = b"alb.ingress.kubernetes.io/listen-ports"
_CSRS = (("obj_ann_begin", ("ann_key", "ann_val")), ("obj_lbi_begin", ("lbi_hostname",)), ("obj_port_begin", ("port_number", "port_proto")))
_FIXED = ("obj_kind", "obj_spec_type", "obj_flags", "obj_ns", "obj_name", "obj_ingress_class")


def _off(refs):
    return (refs & _MASK).astype(np.int64)


def _len(refs):
    return (refs >> np.uint64(40)).astype(np.int64)


def take_rows(cols: dict, rows) -> dict:
    """Object rows `rows` (in that order) of an object column dict; child rows follow their parents, the slab is shared."""
    rows = np.asarray(rows, dtype=np.int64)
    out = {c: np.asarray(cols[c])[rows] for c in _FIXED}
    for bcol, children in _CSRS:
        b = np.asarray(cols[bcol]).astype(np.int64)
        cnt = b[rows + 1] - b[rows]
        nb = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        idx = np.repeat(b[rows] - nb[:-1], cnt) + np.arange(nb[-1], dtype=np.int64)
        out[bcol] = nb.astype(np.uint32)
        for c in children:
            out[c] = np.asarray(cols[c])[idx]
    out["slab"] = cols["slab"]
    return out


def key_is(refs: np.ndarray, slab: np.ndarray, literal: bytes) -> np.ndarray:
    """Mask of the gar_str references whose string equals `literal`."""
    mask = _len(refs) == len(literal)
    cand = np.flatnonzero(mask)
    if len(cand) and literal:
        o = _off(refs[cand])
        same = (slab[o[:, None] + np.arange(len(literal))[None, :]] == np.frombuffer(literal, dtype=np.uint8)[None, :]).all(axis=1)
        mask[cand[~same]] = False
    return mask


def row_keys(cols: dict) -> list:
    """(kind, b"ns/name") of every object row."""
    slab = np.asarray(cols["slab"])
    off, ln = _off(cols["obj_ns"]), _len(cols["obj_ns"]) + 1 + _len(cols["obj_name"])
    raw = slab.tobytes()
    return [(int(k), raw[o:o + n]) for k, o, n in zip(cols["obj_kind"].tolist(), off.tolist(), ln.tolist())]


def compact(cols: dict, new_keys=None) -> dict:
    """A (small) object table with a slab of its own that holds exactly the strings it references.  new_keys[i] (optional,
    bytes "ns/name" or None) renames row i."""
    slab = np.asarray(cols["slab"])
    out = {k: np.array(v, copy=True) for k, v in cols.items() if k != "slab"}
    pieces = []
    renamed = list(new_keys) if new_keys is not None else [None] * len(cols["obj_kind"])
    kb = [nk if nk is not None else k for (_, k), nk in zip(row_keys(cols), renamed)]
    ns_len = [k.index(b"/") if nk is not None else n for k, nk, n in zip(kb, renamed, _len(cols["obj_ns"]).tolist())]
    blob = b"".join(kb)
    koff = np.concatenate([[0], np.cumsum([len(k) for k in kb])]).astype(np.int64)
    nsl = np.asarray(ns_len, dtype=np.int64)
    out["obj_ns"] = (koff[:-1].astype(np.uint64)) | (nsl.astype(np.uint64) << np.uint64(40))
    out["obj_name"] = ((koff[:-1] + nsl + 1).astype(np.uint64)) | ((koff[1:] - koff[:-1] - nsl - 1).astype(np.uint64) << np.uint64(40))
    pieces.append(np.frombuffer(blob, dtype=np.uint8))
    pos = len(blob)
    has_icls = (np.asarray(cols["obj_flags"]) & 2) != 0
    icls = np.where(has_icls, cols["obj_ingress_class"], np.uint64(0)).astype(np.uint64)
    for name, refs in (("obj_ingress_class", icls), ("ann_key", cols["ann_key"]), ("ann_val", cols["ann_val"]), ("lbi_hostname", cols["lbi_hostname"]),
                       ("port_proto", cols["port_proto"])):
        refs = np.asarray(refs, dtype=np.uint64)
        ln = _len(refs)
        loc = np.concatenate([[0], np.cumsum(ln)])[:-1].astype(np.int64)  # where each string starts inside this column's piece
        idx = np.repeat(_off(refs) - loc, ln) + np.arange(int(ln.sum()), dtype=np.int64)
        pieces.append(slab[idx])
        out[name] = (pos + loc).astype(np.uint64) | (ln.astype(np.uint64) << np.uint64(40))
        pos += int(ln.sum())
    out["slab"] = np.concatenate(pieces).astype(np.uint8) if pieces else np.zeros(0, dtype=np.uint8)
    return out


def _pad16(cols: dict) -> dict:
    out = dict(cols)
    s = np.asarray(cols["slab"], dtype=np.uint8)
    out["slab"] = np.concatenate([s, np.zeros((-len(s)) % 16, dtype=np.uint8)])
    return out


class ColumnMirror:
    """The object table after a sequence of deltas, as a column dict laid out like the engine's resident table."""

    def __init__(self, o_cols: dict):
        self.cur = {k: np.array(v, copy=True) for k, v in o_cols.items()}
        self.slab_len = len(self.cur["slab"])
        self.keys = row_keys(self.cur)
        self.rows_of: dict = {}
        for i, k in enumerate(self.keys):
            self.rows_of.setdefault(k, []).append(i)

    def apply(self, up: dict | None, deleted):
        """up: upsert column dict (own slab) or None; deleted: [(kind, "ns/name")].  -> (upsert_row, deleted_row, moved_from)."""
        n = len(self.keys)
        src = {}  # new row -> ("c", current row) | ("u", upsert row), where not the identity
        up_keys = row_keys(up) if up is not None and len(up["obj_kind"]) else []
        del_row, moved, up_row = [], [], []
        keys, rows_of = self.keys, self.rows_of

        def lowest(k):
            rs = rows_of.get(k)
            return min(rs) if rs else GAR_NONE

        for kind, name in deleted:
            k = (int(kind), name.encode("utf-8", "surrogateescape") if isinstance(name, str) else name)
            r = lowest(k)
            del_row.append(r)
            moved.append(GAR_NONE)
            if r == GAR_NONE:
                continue
            last = n - 1
            rows_of[k].remove(r)
            if r != last:
                lk = keys[last]
                rows_of[lk].remove(last)
                rows_of[lk].append(r)
                keys[r] = lk
                src[r] = src.pop(last, ("c", last))
                moved[-1] = last
            else:
                src.pop(last, None)
            keys.pop()
            n -= 1
        for u, k in enumerate(up_keys):
            r = lowest(k)
            if r == GAR_NONE:
                r = n
                n += 1
                keys.append(k)
                rows_of.setdefault(k, []).append(r)
            src[r] = ("u", u)
            up_row.append(r)
        n_cur = len(self.cur["obj_kind"])
        if up_keys:
            both = tables.concat_cols(tables.OBJ_TABLES, ["obj", "ann", "lbi", "port"], [_pad16(self.cur), up])
            self.slab_len = len(_pad16(self.cur)["slab"]) + len(up["slab"])
        else:
            both = self.cur
        sel = np.arange(n, dtype=np.int64)
        for r, (t, i) in src.items():
            sel[r] = i if t == "c" else n_cur + i
        self.cur = take_rows(both, sel)
        self.cur["slab"] = np.asarray(both["slab"])
        return np.array(up_row, dtype=np.uint32), np.array(del_row, dtype=np.uint32), np.array(moved, dtype=np.uint32)

    def compact(self) -> int:
        """The mirror of gar_snapshot_compact(GAR_COMPACT_OBJECTS): the slab holds exactly the live strings.  -> slab_len."""
        self.cur = compact(self.cur)
        self.slab_len = len(self.cur["slab"])
        return self.slab_len

    def snapshot(self, a_cols: dict) -> "tables.Snapshot":
        """A loadable snapshot of the mirrored object table with the given AWS tables."""
        return tables.from_columns(self.cur, a_cols)


def churn(mirror: ColumnMirror, rng: np.random.Generator, frac: float = 0.01, serial: int = 0):
    """One informer-like batch over `frac` of the objects: updates that change decisions (another lbIngress hostname, another
    route53-hostname annotation value, another listen-ports annotation value), 0.05 % adds with fresh keys, 0.05 % deletes.
    -> (upsert column dict with its own slab, [(kind, "ns/name")] deleted keys)."""
    cur = mirror.cur
    n = len(cur["obj_kind"])
    n_add = max(1, int(n * 0.0005))
    n_del = max(1, int(n * 0.0005))
    n_upd = max(1, int(n * frac) - n_add - n_del)
    pick = rng.choice(n, size=min(n, n_upd + n_del), replace=False)
    dels, upd = pick[:n_del], pick[n_del:]
    adds = rng.choice(n, size=n_add, replace=False)
    rows = np.concatenate([upd, adds])
    U = take_rows(cur, rows)
    slab = np.asarray(cur["slab"])
    # the three kinds of decision-changing update, round robin over the updated rows
    lb = np.asarray(cur["obj_lbi_begin"]).astype(np.int64)
    with_lbi = np.flatnonzero(lb[1:] > lb[:-1])
    ub = U["obj_lbi_begin"].astype(np.int64)
    for j in range(0, len(upd), 3):
        if ub[j + 1] > ub[j] and len(with_lbi):
            U["lbi_hostname"][ub[j]] = cur["lbi_hostname"][lb[rng.choice(with_lbi)]]
    ab = U["obj_ann_begin"].astype(np.int64)
    for lit, phase in ((ANN_R53, 1), (ANN_LISTEN, 2)):
        pool = np.asarray(cur["ann_val"])[key_is(np.asarray(cur["ann_key"]), slab, lit)]
        if not len(pool):
            continue
        hit = key_is(U["ann_key"], slab, lit)
        owner = np.searchsorted(ab, np.arange(len(hit)), side="right") - 1
        sel = np.flatnonzero(hit & (owner < len(upd)) & (owner % 3 == phase))
        if len(sel):
            U["ann_val"][sel] = pool[rng.integers(0, len(pool), size=len(sel))]
    keys = row_keys(U)
    new_keys = [None] * len(upd) + [k[:k.index(b"/") + 1] + b"d%d-%d-" % (serial, i) + k[k.index(b"/") + 1:] for i, (_, k) in enumerate(keys[len(upd):])]
    deleted = [(mirror.keys[r][0], mirror.keys[r][1].decode("utf-8", "surrogateescape")) for r in dels.tolist()]
    return compact(U, new_keys), deleted


# ------------------------------------------------------------------ AWS deltas (gar_snapshot_apply_actual)

def take_tree(cols: dict, table: str, rows, out: dict | None = None) -> dict:
    """Rows `rows` (in that order) of an AWS table of an actual column dict, with every table below it (children follow their
    parents, as a load lays them out); string references unchanged."""
    out = {} if out is None else out
    rows = np.asarray(rows, dtype=np.int64)
    for name, kind in tables.ACT_TABLES[table][1]:
        if isinstance(kind, tuple):
            b = np.asarray(cols[name]).astype(np.int64)
            cnt = b[rows + 1] - b[rows]
            nb = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
            idx = np.repeat(b[rows] - nb[:-1], cnt) + np.arange(nb[-1], dtype=np.int64)
            out[name] = nb.astype(np.uint32)
            take_tree(cols, kind[1], idx, out)
        else:
            out[name] = np.asarray(cols[name])[rows]
    return out


def compact_actual(cols: dict) -> dict:
    """An actual column dict with a slab of its own that holds exactly the strings it references."""
    slab = np.asarray(cols["slab"])
    out = {k: np.array(v, copy=True) for k, v in cols.items() if k != "slab"}
    pieces, pos = [], 0
    for t, (_, cl) in tables.ACT_TABLES.items():
        for name, kind in cl:
            if kind != "str":
                continue
            refs = np.asarray(cols[name], dtype=np.uint64)
            if name == "rec_alias_dns":
                refs = np.where(np.asarray(cols["rec_has_alias"]) != 0, refs, np.uint64(0)).astype(np.uint64)
            ln = _len(refs)
            loc = np.concatenate([[0], np.cumsum(ln)])[:-1].astype(np.int64)
            idx = np.repeat(_off(refs) - loc, ln) + np.arange(int(ln.sum()), dtype=np.int64)
            pieces.append(slab[idx])
            out[name] = (pos + loc).astype(np.uint64) | (ln.astype(np.uint64) << np.uint64(40))
            pos += int(ln.sum())
    out["slab"] = np.concatenate(pieces).astype(np.uint8) if pieces else np.zeros(0, dtype=np.uint8)
    return out


def actual_rows(cols: dict, lb_rows=(), acc_rows=(), zone_rows=()) -> dict:
    """A small actual table (the `rows` of an AWS delta, before compact_actual): load balancers `lb_rows`, accelerators
    `acc_rows` with their subtrees and zones `zone_rows` with their record lists, taken from `cols`."""
    out = take_tree(cols, "lb", lb_rows)
    take_tree(cols, "acc", acc_rows, out)
    take_tree(cols, "zone", zone_rows, out)
    out["slab"] = cols["slab"]
    return out


class ActualMirror:
    """The AWS tables after a sequence of AWS deltas, as a column dict laid out like the engine's resident tables (the rules of
    include/garecon.h "AWS deltas"): order preserving, each delta's slab appended at a 16-byte aligned slab_base."""

    def __init__(self, a_cols: dict):
        self.cur = {k: np.array(v, copy=True) for k, v in a_cols.items()}
        self.slab_len = len(self.cur["slab"])

    def sizes(self) -> dict:
        return {nf: len(self.cur[cl[0][0]]) - (1 if isinstance(cl[0][1], tuple) else 0) for t, (nf, cl) in tables.ACT_TABLES.items()}

    def apply(self, rows: dict | None, lb_target=(), acc_target=(), zone_target=(), lb_deleted=(), acc_deleted=()) -> dict:
        """rows: actual column dict with its own slab, or None.  -> the result of the delta: table sizes, slab_base, slab_len."""
        cur = self.cur
        n_rows = {t: len(rows[cl[0][0]]) - (1 if isinstance(cl[0][1], tuple) else 0) for t, (_, cl) in tables.ACT_TABLES.items()} if rows else {}
        has_rows = bool(rows) and (n_rows["lb"] + n_rows["acc"] + n_rows["zone"]) > 0
        base = 0
        both = cur
        if has_rows:
            padded = _pad16(cur)
            base = len(padded["slab"])
            both = tables.concat_cols(tables.ACT_TABLES, ["lb", "acc", "tag", "lis", "pr", "eg", "ep", "rec", "val"], [padded, rows])
            both["zone_name"] = cur["zone_name"]
            both["zone_rec_begin"] = cur["zone_rec_begin"]
        new = {}

        def root(table, nf, target, deleted):
            n = len(cur[nf])
            gone = set(int(r) for r in deleted)
            repl = {int(r): k for k, r in enumerate(target) if int(r) != GAR_NONE}
            sel = [n + repl[r] if r in repl else r for r in range(n) if r not in gone]
            sel += [n + k for k, r in enumerate(target) if int(r) == GAR_NONE]
            take_tree(both, table, np.asarray(sel, dtype=np.int64), new)

        root("lb", "lb_state", lb_target, lb_deleted)
        root("acc", "acc_enabled", acc_target, acc_deleted)
        zb = np.asarray(cur["zone_rec_begin"]).astype(np.int64)
        zrepl = {int(z): k for k, z in enumerate(zone_target)}
        n_rec = int(zb[-1])
        rec_sel = []
        if zrepl:
            rb = np.asarray(rows["zone_rec_begin"]).astype(np.int64)
        for z in range(len(zb) - 1):
            if z in zrepl:
                k = zrepl[z]
                rec_sel.append(np.arange(rb[k], rb[k + 1]) + n_rec)
            else:
                rec_sel.append(np.arange(zb[z], zb[z + 1]))
        cnt = [len(s) for s in rec_sel]
        new["zone_name"] = cur["zone_name"]
        new["zone_rec_begin"] = np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32)
        take_tree(both, "rec", np.concatenate(rec_sel).astype(np.int64) if rec_sel else np.zeros(0, dtype=np.int64), new)
        new["slab"] = np.asarray(both["slab"])
        self.cur = new
        self.slab_len = len(new["slab"])
        out = dict(self.sizes())
        out.pop("n_zones")
        out["slab_base"] = base
        out["slab_len"] = self.slab_len
        return out

    def apply_zones(self, added: dict | None = None, added_at=(), deleted=()) -> dict:
        """The rule of include/garecon.h "zone deltas": for r = 0 .. n_zones, first the new zones with added_at == r in delta
        order, then resident zone r unless it is deleted; records and values follow their zones.  added: an actual column dict
        of zones with their records (own slab, no LB or accelerator rows), or None.  -> the result of the delta: n_zones,
        n_records, n_values, slab_base, slab_len."""
        cur = self.cur
        n = len(cur["zone_name"])
        na = len(added["zone_name"]) if added is not None else 0
        at = np.asarray(added_at, dtype=np.int64).reshape(-1)
        gone = set(np.asarray(deleted, dtype=np.int64).reshape(-1).tolist())
        base, both = 0, cur
        if na:
            padded = _pad16(cur)
            base = len(padded["slab"])
            both = tables.concat_cols(tables.ACT_TABLES, ["rec", "val"], [padded, added])
            zb = np.asarray(cur["zone_rec_begin"]).astype(np.int64)
            both["zone_name"] = np.concatenate([cur["zone_name"], np.asarray(added["zone_name"], dtype=np.uint64) + np.uint64(base)])
            both["zone_rec_begin"] = np.concatenate([zb, np.asarray(added["zone_rec_begin"]).astype(np.int64)[1:] + zb[-1]]).astype(np.uint32)
        sel, k = [], 0
        for r in range(n + 1):
            while k < na and at[k] == r:
                sel.append(n + k)
                k += 1
            if r < n and r not in gone:
                sel.append(r)
        new = {c: v for c, v in cur.items() if c != "slab"}
        take_tree(both, "zone", np.asarray(sel, dtype=np.int64), new)
        new["slab"] = np.asarray(both["slab"])
        self.cur = new
        self.slab_len = len(new["slab"])
        s = self.sizes()
        return {"n_zones": s["n_zones"], "n_records": s["n_records"], "n_values": s["n_values"], "slab_base": base, "slab_len": self.slab_len}

    def apply_records(self, rows: dict | None = None, zone_target=(), rec_at=(), deleted=()) -> dict:
        """The rule of include/garecon.h "record deltas": inside each zone, the delta records placed in front of resident record
        r (rec_at == r) come before r, in delta order, then r unless it is deleted; the ones placed behind the zone's last record
        come last.  Values follow their records; zones, load balancers and accelerators keep their rows.  rows: an actual column
        dict of zones with their records (own slab; zone k stands for resident zone zone_target[k]), or None.  -> the result of
        the delta: n_records, n_values, slab_base, slab_len."""
        cur = self.cur
        zb = np.asarray(cur["zone_rec_begin"]).astype(np.int64)
        n_rec = int(zb[-1])
        at = np.asarray(rec_at, dtype=np.int64).reshape(-1)
        zt = np.asarray(zone_target, dtype=np.int64).reshape(-1)
        gone = np.zeros(n_rec, dtype=bool)
        gone[np.asarray(deleted, dtype=np.int64).reshape(-1)] = True
        base, both = 0, cur
        if len(at):
            padded = _pad16(cur)
            base = len(padded["slab"])
            both = tables.concat_cols(tables.ACT_TABLES, ["rec", "val"], [padded, rows])
        # one sort key per placed record: (zone, position, inserts before the resident record at the same position, delta order)
        res = np.flatnonzero(~gone)
        res_zone = np.searchsorted(zb, res, side="right") - 1
        ub = np.asarray(rows["zone_rec_begin"]).astype(np.int64) if len(at) else np.zeros(1, dtype=np.int64)
        ins_zone = np.repeat(zt[:len(ub) - 1], ub[1:] - ub[:-1]) if len(at) else np.zeros(0, dtype=np.int64)
        zone = np.concatenate([res_zone, ins_zone])
        pos = np.concatenate([res, at])
        tie = np.concatenate([np.ones(len(res), dtype=np.int64), np.zeros(len(at), dtype=np.int64)])
        src = np.concatenate([res, n_rec + np.arange(len(at), dtype=np.int64)])
        order = np.lexsort((src, tie, pos, zone))
        new = {c: v for c, v in cur.items() if c != "slab"}
        new["zone_rec_begin"] = np.concatenate([[0], np.cumsum(np.bincount(zone, minlength=len(zb) - 1))]).astype(np.uint32)
        take_tree(both, "rec", src[order], new)
        new["slab"] = np.asarray(both["slab"])
        self.cur = new
        self.slab_len = len(new["slab"])
        s = self.sizes()
        return {"n_records": s["n_records"], "n_values": s["n_values"], "slab_base": base, "slab_len": self.slab_len}

    def compact(self) -> int:
        """The mirror of gar_snapshot_compact(GAR_COMPACT_ACTUAL): the slab holds exactly the live strings.  -> slab_len."""
        self.cur = compact_actual(self.cur)
        self.slab_len = len(self.cur["slab"])
        return self.slab_len

    def snapshot(self, o_cols: dict) -> "tables.Snapshot":
        """A loadable snapshot of the given object table with the mirrored AWS tables."""
        return tables.from_columns(o_cols, self.cur)


def aws_churn(mirror: ActualMirror, rng: np.random.Generator, frac: float = 0.01, max_zones: int = 4):
    """One re-list batch over `frac` of the AWS rows, like the lists a worker re-issues after executing a batch: load balancer
    state flips plus a few appended (duplicate (region, name)) and deleted LBs; accelerator subtrees rewritten (a tag value,
    listener ports, endpoints), a few accelerators appended (copies) and deleted; the record lists of up to `max_zones` zones
    replaced (a record dropped, another repeated).  -> keyword arguments of Engine.apply_actual / ActualMirror.apply, with
    rows = a compact actual column dict."""
    cur = mirror.cur
    n_lb, n_acc, n_zone = len(cur["lb_state"]), len(cur["acc_enabled"]), len(cur["zone_name"])

    def split(n, k_change, k_del):
        pick = rng.choice(n, size=min(n, k_change + k_del), replace=False) if n else np.zeros(0, dtype=np.int64)
        return np.sort(pick[k_del:]), np.sort(pick[:k_del])

    lb_upd, lb_del = split(n_lb, max(1, int(n_lb * frac)), max(1, int(n_lb * frac / 20)) if n_lb > 2 else 0)
    lb_add = rng.choice(n_lb, size=max(1, int(n_lb * frac / 20)), replace=True) if n_lb else np.zeros(0, dtype=np.int64)
    acc_upd, acc_del = split(n_acc, max(1, int(n_acc * frac)), max(1, int(n_acc * frac / 20)) if n_acc > 2 else 0)
    acc_add = rng.choice(n_acc, size=max(1, int(n_acc * frac / 20)), replace=True) if n_acc else np.zeros(0, dtype=np.int64)
    zones = np.sort(rng.choice(n_zone, size=min(n_zone, max_zones), replace=False)) if n_zone else np.zeros(0, dtype=np.int64)
    rows = actual_rows(cur, np.concatenate([lb_upd, lb_add]), np.concatenate([acc_upd, acc_add]), zones)
    # load balancers: state flips on the re-described rows, another row's DNS name on the appended copies
    st = rows["lb_state"]
    st[:len(lb_upd)] = np.where(st[:len(lb_upd)] == 0, 1, 0)
    if len(lb_add):
        rows["lb_dns"][len(lb_upd):] = cur["lb_dns"][rng.integers(0, n_lb, size=len(lb_add))]
    # accelerator subtrees: a tag value, listener ports and endpoints taken from elsewhere in the batch
    if len(rows["tag_val"]):
        t = rng.random(len(rows["tag_val"])) < 0.2
        rows["tag_val"][t] = rows["tag_val"][rng.integers(0, len(rows["tag_val"]), size=int(t.sum()))]
    if len(rows["pr_from"]):
        p = rng.random(len(rows["pr_from"])) < 0.3
        rows["pr_from"][p] = rng.choice(np.array([80, 443, 8080, 53], dtype=np.int32), size=int(p.sum()))
    if len(rows["ep_id"]):
        rows["ep_id"] = rows["ep_id"][rng.permutation(len(rows["ep_id"]))]
    # record lists: per zone, one record dropped and another one repeated
    zb = rows["zone_rec_begin"].astype(np.int64)
    keep = []
    for k in range(len(zones)):
        recs = list(range(zb[k], zb[k + 1]))
        if recs and rng.random() < 0.7:
            recs.pop(int(rng.integers(0, len(recs))))
        if recs and rng.random() < 0.5:
            recs.append(recs[int(rng.integers(0, len(recs)))])
        keep.append(recs)
    rec_rows = take_tree(rows, "rec", np.asarray([r for rs in keep for r in rs], dtype=np.int64))
    rows.update(rec_rows)
    rows["zone_rec_begin"] = np.concatenate([[0], np.cumsum([len(rs) for rs in keep])]).astype(np.uint32)
    return dict(rows=compact_actual(rows),
                lb_target=np.concatenate([lb_upd, np.full(len(lb_add), GAR_NONE)]).astype(np.uint32),
                acc_target=np.concatenate([acc_upd, np.full(len(acc_add), GAR_NONE)]).astype(np.uint32),
                zone_target=zones.astype(np.uint32), lb_deleted=lb_del.astype(np.uint32), acc_deleted=acc_del.astype(np.uint32))


def zone_churn(mirror: ActualMirror, rng: np.random.Generator, n_add: int = 10, rec_frac: float = 0.01, n_del: int = 0, serial: int = 0):
    """One change of the hosted-zone set, as a worker sees it between two ListHostedZones answers: `n_del` random zones deleted
    and `n_add` zones created at random rows, whose record sets total about `rec_frac` of all records.  With n_add >= 2, the
    first new zone is a subzone of the zone with the most records, named after one of its record names and holding that
    name's record sets (so the hostname resolves to the subzone from now on), and the second repeats the name of a resident
    zone, listed in front of it (so it wins the zone walk), with half of that zone's records.  The others get fresh names and
    a run of records copied from a random record row on (across zone boundaries).  -> keyword arguments of Engine.apply_zones / ActualMirror.apply_zones, with
    added = a compact actual column dict."""
    cur = mirror.cur
    slab = np.asarray(cur["slab"])
    n = len(cur["zone_name"])
    zb = np.asarray(cur["zone_rec_begin"]).astype(np.int64)
    n_rec = int(zb[-1])
    budget = int(n_rec * rec_frac)
    recs, names, at = [], [], []  # per new zone: record rows of `cur`, zone name (gar_str into cur's slab, or fresh bytes), row
    if n_add >= 2 and n and n_rec:
        z = int(np.argmax(zb[1:] - zb[:-1]))
        r = int(rng.integers(zb[z], zb[z + 1]))
        nm = slab[int(_off(cur["rec_name"][r:r + 1])[0]):][:int(_len(cur["rec_name"][r:r + 1])[0])].tobytes()
        recs.append(zb[z] + np.flatnonzero(key_is(np.asarray(cur["rec_name"][zb[z]:zb[z + 1]]), slab, nm)))
        names.append(cur["rec_name"][r])
        at.append(int(rng.integers(0, n + 1)))
        d = int(rng.integers(0, n))
        recs.append(np.arange(zb[d], zb[d] + min((zb[d + 1] - zb[d]) // 2, max(0, budget // 3))))
        names.append(cur["zone_name"][d])
        at.append(d)
    left = max(0, budget - sum(len(x) for x in recs))
    n_fresh = n_add - len(recs)
    for i in range(n_fresh):
        take = min(n_rec, left // n_fresh + (1 if i < left % n_fresh else 0))
        lo = int(rng.integers(0, n_rec - take + 1))
        recs.append(np.arange(lo, lo + take))  # a run of record rows, across zone boundaries
        names.append(b"zc%d-%d.churn.test." % (serial, i))
        at.append(int(rng.integers(0, n + 1)))
    order = np.argsort(np.asarray(at, dtype=np.int64), kind="stable")
    rows = actual_rows(cur)
    rec_rows = np.concatenate([recs[k] for k in order]).astype(np.int64) if len(order) else np.zeros(0, dtype=np.int64)
    rows.update(take_tree(cur, "rec", rec_rows))
    rows["zone_rec_begin"] = np.concatenate([[0], np.cumsum([len(recs[k]) for k in order])]).astype(np.uint32)
    rows["zone_name"] = np.asarray([0 if isinstance(names[k], bytes) else names[k] for k in order], dtype=np.uint64)
    added = compact_actual(rows)
    fresh = [(i, names[k]) for i, k in enumerate(order) if isinstance(names[k], bytes)]
    if fresh:
        pos = len(added["slab"])
        for i, nm in fresh:
            added["zone_name"][i] = np.uint64(pos) | (np.uint64(len(nm)) << np.uint64(40))
            pos += len(nm)
        added["slab"] = np.concatenate([added["slab"], np.frombuffer(b"".join(nm for _, nm in fresh), dtype=np.uint8)])
    deleted = np.sort(rng.choice(n, size=min(n, n_del), replace=False)) if n_del and n else np.zeros(0, dtype=np.int64)
    return dict(added=added, added_at=np.asarray(at, dtype=np.uint32)[order], deleted=deleted.astype(np.uint32))


def largest_zones_deleted(mirror: ActualMirror, k: int = 10):
    """A zone delta that deletes the `k` zones with the most records.  -> keyword arguments of Engine.apply_zones /
    ActualMirror.apply_zones (added = None)."""
    zb = np.asarray(mirror.cur["zone_rec_begin"]).astype(np.int64)
    rows = np.sort(np.argsort(-(zb[1:] - zb[:-1]), kind="stable")[:k])
    return dict(added=None, added_at=np.zeros(0, dtype=np.uint32), deleted=rows.astype(np.uint32))


def actual_struct(cols: dict):
    """(Snapshot owning the buffers, its GarActual) for an actual column dict: the `rows` of Engine.apply_actual."""
    empty_objects = {c: np.zeros(0 if not isinstance(k, tuple) else 1, dtype=np.uint32 if isinstance(k, tuple) else tables._DT[k])
                     for t, (_, cl) in tables.OBJ_TABLES.items() for c, k in cl}
    empty_objects["slab"] = np.zeros(0, dtype=np.uint8)
    snap = tables.from_columns(empty_objects, cols)
    return snap, snap.actual


def objects_struct(cols: dict):
    """(Snapshot owning the buffers, its GarObjects) for an object column dict: the `upserts` of Engine.apply_objects."""
    empty_actual = {c: np.zeros(0 if not isinstance(k, tuple) else 1, dtype=np.uint32 if isinstance(k, tuple) else tables._DT[k])
                    for t, (_, cl) in tables.ACT_TABLES.items() for c, k in cl}
    empty_actual["slab"] = np.zeros(0, dtype=np.uint8)
    snap = tables.from_columns(cols, empty_actual)
    return snap, snap.objects


# ------------------------------------------------------------------ record deltas (gar_snapshot_apply_records)

def record_rows(cols: dict, zones, placed) -> dict:
    """The `rows` of a record delta: zones `zones` (ascending resident zone rows of `cols`) with, per zone, the records `placed[k]`
    (record rows of `cols`, in delta order), as a compact actual column dict with its own slab."""
    rows = actual_rows(cols)
    rows["zone_name"] = np.asarray(cols["zone_name"], dtype=np.uint64)[np.asarray(zones, dtype=np.int64)]
    rec = np.asarray([r for rs in placed for r in rs], dtype=np.int64)
    rows.update(take_tree(cols, "rec", rec))
    rows["zone_rec_begin"] = np.concatenate([[0], np.cumsum([len(rs) for rs in placed])]).astype(np.uint32)
    return compact_actual(rows)


def record_churn(mirror: ActualMirror, rng: np.random.Generator, n_zones: int = 8, per_zone: int = 3):
    """One batch of record-set edits inside resident zones, as a worker re-describes them: in `n_zones` random zones (and in the
    first run of adjacent empty zones, when there is one) record sets replaced in place (alias target or values taken from
    another record of the table), inserted at the zone's front, at its end and in between (copies of records from anywhere), and
    deleted; now and then every record of a zone deleted.  -> keyword arguments of Engine.apply_records /
    ActualMirror.apply_records, with rows = a compact actual column dict."""
    cur = mirror.cur
    zb = np.asarray(cur["zone_rec_begin"]).astype(np.int64)
    nz, n_rec = len(zb) - 1, int(zb[-1])
    if not nz:
        return dict(rows=None, zone_target=np.zeros(0, dtype=np.uint32), rec_at=np.zeros(0, dtype=np.uint32), deleted=np.zeros(0, dtype=np.uint32))
    zones = set(rng.choice(nz, size=min(nz, n_zones), replace=False).tolist())
    empty = np.flatnonzero(zb[1:] == zb[:-1])
    adj = empty[np.flatnonzero(empty[1:] == empty[:-1] + 1)] if len(empty) > 1 else empty[:0]
    if len(adj):
        zones.update([int(adj[0]), int(adj[0]) + 1])
    elif len(empty):
        zones.add(int(empty[0]))
    alias = np.flatnonzero(np.asarray(cur["rec_has_alias"]) != 0)
    extra = {}  # delta record -> (column, value) overrides, applied after the records are taken
    targets, placed, at, deleted = [], [], [], []
    for z in sorted(zones):
        a, b = int(zb[z]), int(zb[z + 1])
        ins = []  # (rec_at, source record row, override or None)
        if b > a and rng.random() < 0.1:
            deleted.extend(range(a, b))  # the zone's every record set deleted ...
            if rng.random() < 0.5 and n_rec:
                ins.append((b, int(rng.integers(0, n_rec)), None))  # ... and one listed again behind them
        else:
            for r in (rng.choice(np.arange(a, b), size=min(b - a, per_zone), replace=False).tolist() if b > a else []):
                c = rng.random()
                if c < 0.4:  # replaced: the same set with another alias target or another record's values
                    deleted.append(r)
                    if cur["rec_has_alias"][r] and len(alias):
                        ins.append((r, r, ("rec_alias_dns", cur["rec_alias_dns"][int(rng.choice(alias))])))
                    else:
                        ins.append((r, r, ("values", int(rng.integers(0, n_rec)))))
                elif c < 0.7:
                    deleted.append(r)
                else:
                    ins.append((r, int(rng.integers(0, n_rec)), None))  # inserted in front of r
            if n_rec:
                ins.append((a, int(rng.integers(0, n_rec)), None))  # at the front (in an empty zone: its only record)
                ins.append((b, int(rng.integers(0, n_rec)), None))  # at the end
        if not ins:
            continue
        ins.sort(key=lambda x: x[0])
        base = sum(len(p) for p in placed)
        for k, (_, _, o) in enumerate(ins):
            if o is not None:
                extra[base + k] = o
        targets.append(z)
        placed.append([s for _, s, _ in ins])
        at.extend(x for x, _, _ in ins)
    if not targets:
        return dict(rows=None, zone_target=np.zeros(0, dtype=np.uint32), rec_at=np.zeros(0, dtype=np.uint32), deleted=np.asarray(sorted(set(deleted)), dtype=np.uint32))
    rows = actual_rows(cur)
    rows["zone_name"] = np.asarray(cur["zone_name"], dtype=np.uint64)[np.asarray(targets, dtype=np.int64)]
    src = [s for p in placed for s in p]
    for k, (col, v) in extra.items():
        if col == "values":
            src[k] = src[k], v  # the record of src[k] with the values of record v
    recs = [s if isinstance(s, int) else s[0] for s in src]
    rows.update(take_tree(cur, "rec", np.asarray(recs, dtype=np.int64)))
    vb = np.asarray(cur["rec_val_begin"]).astype(np.int64)
    vals = [np.arange(vb[s], vb[s + 1]) if isinstance(s, int) else np.arange(vb[s[1]], vb[s[1] + 1]) for s in src]
    rows["rec_val_begin"] = np.concatenate([[0], np.cumsum([len(v) for v in vals])]).astype(np.uint32)
    rows["val_value"] = np.asarray(cur["val_value"])[np.concatenate(vals).astype(np.int64)] if vals else np.zeros(0, dtype=np.uint64)
    for k, (col, v) in extra.items():
        if col == "rec_alias_dns":
            rows["rec_alias_dns"][k] = v
    rows["zone_rec_begin"] = np.concatenate([[0], np.cumsum([len(p) for p in placed])]).astype(np.uint32)
    return dict(rows=compact_actual(rows), zone_target=np.asarray(targets, dtype=np.uint32), rec_at=np.asarray(at, dtype=np.uint32),
                deleted=np.asarray(sorted(set(deleted)), dtype=np.uint32))


def record_refresh(resident: dict, cloud: dict, rec_rows) -> dict:
    """The record delta that re-describes the resident record rows `rec_rows` from the cloud's tables (actual column dicts with
    the same zone table): per row, ListResourceRecordSets(zone, StartRecordName = its name, StartRecordType = its type,
    MaxItems = 1) — the cloud's set of that (zone, name, type) replaces the row in place, or the row is deleted when the cloud has
    none.  The n-th resident row of a (zone, name, type) maps to the n-th cloud set of it.  -> keyword arguments of
    Engine.apply_records / ActualMirror.apply_records."""
    def ids(cols):
        zb = np.asarray(cols["zone_rec_begin"]).astype(np.int64)
        slab = np.asarray(cols["slab"]).tobytes()
        name, typ = np.asarray(cols["rec_name"]), np.asarray(cols["rec_type"])
        out, seen = [], {}
        for z in range(len(zb) - 1):
            for r in range(zb[z], zb[z + 1]):
                o, n = int(name[r]) & ((1 << 40) - 1), int(name[r]) >> 40
                key = (z, slab[o:o + n], int(typ[r]))
                seen[key] = seen.get(key, -1) + 1
                out.append(key + (seen[key],))
        return out
    rid, cid = ids(resident), ids(cloud)
    where = {k: r for r, k in enumerate(cid)}
    rows = sorted(set(int(r) for r in rec_rows))
    zb = np.asarray(resident["zone_rec_begin"]).astype(np.int64)
    by_zone = {}
    for r in rows:
        c = where.get(rid[r])
        if c is not None:
            by_zone.setdefault(rid[r][0], []).append((r, c))
    zones = sorted(by_zone)
    d = record_rows(cloud, zones, [[c for _, c in by_zone[z]] for z in zones]) if zones else None
    return dict(rows=d, zone_target=np.asarray(zones, dtype=np.uint32), rec_at=np.asarray([r for z in zones for r, _ in by_zone[z]], dtype=np.uint32),
                deleted=np.asarray(rows, dtype=np.uint32))


def record_redescribe(cols: dict, rec_rows) -> dict:
    """The record delta a worker applies after re-describing the resident record rows `rec_rows` and finding them as `cols` (the
    mirror of the resident tables) holds them: each row replaced in place by its own set (a delete of the row plus an insert in
    front of it).  -> keyword arguments of Engine.apply_records / ActualMirror.apply_records."""
    rows = np.unique(np.asarray(rec_rows, dtype=np.int64).reshape(-1))
    zb = np.asarray(cols["zone_rec_begin"]).astype(np.int64)
    zones, counts = np.unique(np.searchsorted(zb, rows, side="right") - 1, return_counts=True)
    d = actual_rows(cols)
    d["zone_name"] = np.asarray(cols["zone_name"], dtype=np.uint64)[zones]
    d.update(take_tree(cols, "rec", rows))
    d["zone_rec_begin"] = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    return dict(rows=compact_actual(d), zone_target=zones.astype(np.uint32), rec_at=rows.astype(np.uint32), deleted=rows.astype(np.uint32))
