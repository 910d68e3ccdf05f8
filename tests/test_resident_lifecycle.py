"""The resident snapshot's whole call surface in one process: object, AWS and zone deltas (small and large batches), slab
compactions, refused deltas and deletes at scan-tile edges, in random sequences on the adversarial clusters of
tests/scalemodels.py.  After every step each answer is checked against its arbiter on mirrors of the resident tables: the full
diff and gar_diff_keys against the oracle, gar_bindings_diff against the oracle, the device-resident result against gar_diff
byte for byte, gar_read_set against tests/readset_ref.py, and gar_snapshot_export against the numpy compaction of the mirrors
(restored into a second engine every few steps).  Every few steps the read set is also shown sufficient after the deltas: a
second engine loaded from the export gets every AWS row outside the set rewritten and must answer gar_diff_keys as the main
engine does.  On the GPU the recorded-launch rules of tests/test_launch_replay.py hold throughout, and an engine created with
GAR_NO_GRAPH=1 gives the same full diffs on the same schedule.

At 2*10^4 objects every table a delta re-lays (objects, lbIngress rows, accelerators, tags, records, values) spans more than
four 2048-item scan tiles, so the splice's scans, its row remap and the child relayout cross tile and block edges with hot keys,
duplicate load balancers, several lbIngress rows per object and orphans in the tables.  The host simulation runs the same
state machine at about 10^3 objects."""
import bisect
import copy
import os
import random
from collections import Counter

import numpy as np
import pytest

import egbcases
import readset_ref
import scalemodels
from test_launch_replay import _engine, _same_results
from test_object_deltas import Events, Mirror, assert_same_full, key_of
from test_actual_deltas import AwsEvents
from test_read_set import apply_rows, got as read_set_got, rewrite_outside
from test_snapshot_export import check_export
from test_zone_deltas import State, ZoneEvents

OBJ, ACT, BOTH = 1, 2, 3
NONE = 0xFFFFFFFF
TILE = 2048  # items per tile of the backend's exclusive_scan (gar_engine.cu SCAN_TILE)
EDGES = (TILE - 1, TILE, 2 * TILE - 1, 2 * TILE)
THREADS = os.cpu_count() or 4
MUTATIONS = ("obj_small", "obj_1pct", "obj_10pct", "aws_small", "aws_large", "zones", "compact", "refused", "edge_rows", "edge_tile", "edge_aws")
QUERIES = ("full", "keys", "bindings", "device", "read_set", "export", "restore", "sufficiency")
LEVELS = ("objects", "lbi", "accs", "tags", "records", "values")  # the spliced levels that must exceed four scan tiles at scale


class FastMirror(Mirror):
    """test_object_deltas.Mirror with the lowest row of each key kept in an index, so that batches of 10^3 keys over 10^4
    rows stay quick.  The same rules: deletes first (the last row moves into the freed one), then upserts (lowest row of the key
    replaced, or appended)."""

    def __init__(self, objects, snap):
        super().__init__(objects, snap)
        self.rows = {}
        for r, ob in enumerate(self.objects):
            self.rows.setdefault(key_of(ob), []).append(r)

    def _lowest(self, k):
        rs = self.rows.get(k)
        return rs[0] if rs else NONE

    def _move(self, k, old, new):
        rs = self.rows[k]
        rs.remove(old)
        if new != NONE:
            bisect.insort(rs, new)
        if not rs:
            del self.rows[k]

    def apply(self, upserts, deleted, upsert_snap=None):
        deleted_row, moved_from, upsert_row = [], [], []
        for k in deleted:
            r = self._lowest(k)
            last = len(self.objects) - 1
            deleted_row.append(r)
            moved_from.append(NONE if r in (NONE, last) else last)
            if r != NONE:
                self._move(k, r, NONE)
                if r != last:
                    self._move(key_of(self.objects[last]), last, r)
                self.objects[r] = self.objects[last]
                self.objects.pop()
        for ob in upserts:
            k = key_of(ob)
            r = self._lowest(k)
            if r == NONE:
                r = len(self.objects)
                self.objects.append(ob)
                self.rows[k] = [r]
            else:
                self.objects[r] = ob
            upsert_row.append(r)
        base = 0
        if upserts:
            base = (len(self.slab) + 15) & ~15
            self.slab += b"\0" * (base - len(self.slab))
            self.slab += upsert_snap.arrays["o.slab"][:int(upsert_snap.objects.slab_len)].tobytes()
        return upsert_row, deleted_row, moved_from, base


def make_model(name, seed, n):
    """-> (objects, actual, keys of objects dropped from the cache, bindings, known endpoint groups)."""
    dropped = []
    if name == "rand":
        objects, actual, dropped = scalemodels.randmodel_dropped(seed, n)
    elif name == "hot":
        objects, actual = scalemodels.hot_cluster(seed, n)
    elif name == "multilbi":
        objects, actual = scalemodels.multilbi_cluster(seed, n)
    elif name == "bindings":
        objects, actual, bindings, known = scalemodels.bindings_cluster(seed, n, 3 * n)
        return objects, actual, dropped, bindings, known
    else:
        raise KeyError(name)
    _, _, bindings, known = egbcases.random_bindings(seed, n_objects=n, n_bindings=n)  # names the randmodel objects of this seed
    return objects, actual, dropped, bindings, known


def _counts(actual):
    accs = actual["accelerators"]
    recs = [r for z in actual["zones"] for r in z.get("records", [])]
    return {"accs": len(accs), "tags": sum(len(a.get("tags", [])) for a in accs), "records": len(recs),
            "values": sum(len(r.get("values", [])) for r in recs)}


class Lifecycle:
    """One engine with its mirrors (test_zone_deltas.State: objects, the AwsModel dict model and deltas.ActualMirror) and the
    mutations and queries of the state machine.  check=False (the GAR_NO_GRAPH control) runs the same calls without the
    arbiters; `schedule` then gives the number of full diffs after each step."""

    def __init__(self, garecon, oracle, engine, second, name, seed, n, gpu, check=True, schedule=None):
        self.g, self.oracle, self.e, self.e2, self.gpu, self.check = garecon, oracle, engine, second, gpu, check
        objects, actual, self.dropped, bindings, known = make_model(name, seed, n)
        self.b = garecon.pack_bindings(bindings, known)
        self.s = State(garecon, oracle, engine, objects, actual, oracle_mode=1)
        self.s.om = FastMirror(objects, self.s.snap)
        self.oev, self.aev, self.zev = Events(seed, actual), AwsEvents(seed), ZoneEvents(seed)
        self.rng = random.Random(seed * 7 + 11)
        self.gone = set()  # keys this run's deltas deleted (and that are not back)
        self.keep = []  # packed deltas and exports: the host simulation reads columns in place
        self.schedule = list(schedule) if schedule is not None else None
        self.counts, self.results, self.modes = [], [], []
        self.seen = Counter()
        self.spliced = Counter()

    # ------------------------------------------------------------------ mutations
    def _objects(self, upserts, deleted):
        usnap = self.g.pack(upserts, None) if upserts else None
        self.keep.append(usnap)
        res = self.e.apply_objects(usnap.objects if usnap else None, deleted)
        up_row, del_row, moved, base = self.s.om.apply(upserts, deleted, usnap)
        assert res.upsert_row.tolist() == up_row and res.deleted_row.tolist() == del_row and res.moved_from.tolist() == moved
        assert res.n_objects == len(self.s.om.objects) and res.slab_len == len(self.s.om.slab)
        if upserts:
            assert res.slab_base == base
        present = set(self.s.om.rows)
        self.gone = {k for k in self.gone | set(deleted) if k not in present}
        self.spliced["objects"] = max(self.spliced["objects"], int(res.n_objects))
        self.spliced["lbi"] = max(self.spliced["lbi"], sum(len(o.get("lb_ingress", [])) for o in self.s.om.objects))

    def _aws(self, d):
        self.s.aws(d)
        self.keep.append(d)
        c = _counts(self.s.model.actual)
        if d.get("accs") or d.get("acc_deleted"):
            for k in ("accs", "tags"):
                self.spliced[k] = max(self.spliced[k], c[k])
        if d.get("zones"):
            for k in ("records", "values"):
                self.spliced[k] = max(self.spliced[k], c[k])

    def _zones(self, added, deleted):
        self.s.zones(added, deleted)
        c = _counts(self.s.model.actual)
        for k in ("records", "values"):
            self.spliced[k] = max(self.spliced[k], c[k])

    def large_objects(self, frac):
        """About frac of the rows, from Events' own pieces: in-place updates, deletes of keys that own accelerators and records,
        adds with fresh keys and adds that adopt orphaned owners; each key at most once."""
        ev, rng, objects = self.oev, self.oev.rng, self.s.om.objects
        k = max(4, int(len(objects) * frac))
        present = set(self.s.om.rows)
        used, upserts = set(), []
        owning = [x for x in ev.owner_keys if x in present]
        deleted = rng.sample(owning, min(len(owning), k // 4))
        used.update(deleted)
        for ob in rng.sample(objects, min(len(objects), k // 2)):
            ob = ev._update(ob, objects)
            if key_of(ob) not in used:
                used.add(key_of(ob))
                upserts.append(ob)
        for _ in range(k // 8):
            ev.serial += 1
            ob = copy.deepcopy(rng.choice(ev.pool))
            ob["name"] = f"add{ev.serial}-{ob['name']}"
            used.add(key_of(ob))
            upserts.append(ob)
        absent = [x for x in ev.owner_keys if x not in present and x not in used]
        for x in rng.sample(absent, min(len(absent), k // 8)):
            base = [o for o in ev.pool if o.get("kind", "service") == ("service" if x[0] == 0 else "ingress")]
            if base:
                ob = copy.deepcopy(rng.choice(base))
                ob["ns"], ob["name"] = x[1].split("/", 1)
                used.add(x)
                upserts.append(ob)
        rng.shuffle(upserts)
        self._objects(upserts, deleted)

    def large_aws(self, frac):
        """AwsEvents' kinds over about frac of the rows (at least hundreds): LB replaces and deletes (rows ahead of a duplicate
        (region, name) first), appended duplicates; accelerator subtrees replaced, appended and deleted; record lists replaced.
        Replaced and deleted rows never overlap."""
        a, rng, aev = self.s.model.actual, self.aev.rng, self.aev
        lbs, accs, zones = a["lbs"], a["accelerators"], a["zones"]
        d = {"lbs": [], "accs": [], "zones": [], "lb_deleted": [], "acc_deleted": []}
        later = Counter((lb["region"], lb["name"]) for lb in lbs)
        ahead = []
        for r, lb in enumerate(lbs):
            later[lb["region"], lb["name"]] -= 1
            if later[lb["region"], lb["name"]] > 0:
                ahead.append(r)  # a row with a duplicate (region, name) behind it
        k = min(len(lbs), max(200, int(len(lbs) * frac)))
        dels = set(rng.sample(ahead, min(len(ahead), k // 3)))
        rows = [r for r in rng.sample(range(len(lbs)), k) if r not in dels]
        for r in rows[:len(rows) // 2]:
            dels.add(r)
        for r in rows[len(rows) // 2:]:
            lb = dict(lbs[r], state=rng.choice(["active", "provisioning", "failed", "active_impaired"]))
            if rng.random() < 0.3:
                lb["dns"] = rng.choice(lbs)["dns"]
            d["lbs"].append((r, lb))
        d["lb_deleted"] = sorted(dels)
        rng.shuffle(d["lb_deleted"])
        for _ in range(k // 10):
            d["lbs"].append((NONE, dict(rng.choice(lbs), dns="dup-" + rng.choice(lbs)["dns"], state=rng.choice(["active", "provisioning"]))))
        k = min(len(accs), max(200, int(len(accs) * frac)))
        rows = rng.sample(range(len(accs)), k)
        d["acc_deleted"] = rows[:k // 3]
        for r in rows[k // 3:]:
            if rng.random() < 0.5:
                new = copy.deepcopy(accs[r])  # the same accelerator, re-described after the worker changed it
                for li in new.get("listeners", []):
                    li["ports"] = [rng.choice([80, 443, 8080])] + li.get("ports", [])[1:]
                    for eg in li.get("egs", []):
                        eg["endpoints"] = rng.sample([x["arn"] for x in lbs], min(len(lbs), rng.randrange(0, 3)))
            else:
                new = copy.deepcopy(rng.choice(aev.acc_pool + [accs[rng.randrange(len(accs))]]))
            d["accs"].append((r, new))
        for _ in range(k // 10):
            d["accs"].append((NONE, copy.deepcopy(rng.choice(accs + aev.acc_pool))))
        for z in rng.sample(range(len(zones)), min(len(zones), 2)):
            recs = copy.deepcopy(zones[z].get("records", []))
            rng.shuffle(recs)
            recs = recs[:len(recs) - len(recs) // 10]
            recs.append({"name": f"txt{rng.randrange(99)}.{zones[z]['name']}", "type": "TXT", "values": [f'"v{i}"' for i in range(rng.randrange(2, 40))]})
            d["zones"].append((z, recs))
        self._aws(d)

    def edge_rows(self):
        """Delete the objects at rows 2047, 2048, 4095 and 4096 (a few rows at the ends of a small table)."""
        objects = self.s.om.objects
        rows = [r for r in EDGES if r < len(objects)] or [0, len(objects) // 2, len(objects) - 1]
        keys = list(dict.fromkeys(key_of(objects[r]) for r in rows))
        self._objects([], keys)

    def edge_tile(self):
        """Delete every object row of the second scan tile (rows 2048-4095; a quarter of a small table)."""
        objects = self.s.om.objects
        lo, hi = (TILE, 2 * TILE) if len(objects) > 2 * TILE + 100 else (len(objects) // 4, len(objects) // 2)
        keys = list(dict.fromkeys(key_of(objects[r]) for r in range(lo, hi)))
        self._objects([], keys)

    def edge_aws(self):
        """LB and accelerator rows at the same edges deleted; accelerator subtrees of another shape next to them, so the child
        CSR levels (tags, listeners, port ranges, endpoint groups, endpoints) are re-laid across the edges too."""
        a = self.s.model.actual
        nl, na = len(a["lbs"]), len(a["accelerators"])
        lrows = [r for r in EDGES if r < nl] or [0, nl // 2, nl - 1]
        arows = [r for r in EDGES if r < na] or [0, na // 2, na - 1]
        near = [r for r in (EDGES[0] - 1, EDGES[2] - 1, EDGES[3] + 1) if r < na and r not in arows] or [na // 2 + 1]
        d = {"lbs": [], "accs": [(r, copy.deepcopy(self.aev.acc_pool[k % len(self.aev.acc_pool)])) for k, r in enumerate(near) if r < na and r not in arows],
             "zones": [], "lb_deleted": sorted(set(lrows)), "acc_deleted": sorted(set(arows))}
        self._aws(d)

    def refused(self):
        g, e, rng = self.g, self.e, self.rng
        c = rng.randrange(4)
        with pytest.raises(g.GarError) as ei:
            if c == 0:
                e.apply_objects(None, [key_of(self.s.om.objects[rng.randrange(len(self.s.om.objects))])] * 2)  # the same key twice
            elif c == 1:
                r = rng.randrange(len(self.s.model.actual["accelerators"]))
                e.apply_actual(acc_deleted=[r, r])  # the same row twice
            elif c == 2:
                rows = g.pack([], {"lbs": self.s.model.actual["lbs"][:1]})
                self.keep.append(rows)
                e.apply_actual(rows.actual, lb_target=[0], lb_deleted=[0])  # one row replaced and deleted
            else:
                e.apply_zones(None, [], [0, 0])  # a zone row twice
        assert ei.value.rc == g.abi.GAR_E_INVALID

    def compact(self):
        groups = self.rng.choice([OBJ, ACT, BOTH])
        res = self.e.compact(groups)
        if groups & OBJ:
            self.s.om.slab = bytearray(self.e.read_slab(OBJ, 0, res.obj_slab_len).tobytes())
        if groups & ACT:
            self.s.model.slab_len = int(res.act_slab_len)
            assert int(res.act_slab_len) == self.s.am.compact()

    def mutate(self, kind):
        self.seen[kind] += 1
        if kind == "obj_small":
            self._objects(*self.oev.batch(self.s.om.objects))
        elif kind == "obj_1pct":
            self.large_objects(0.01)
        elif kind == "obj_10pct":
            self.large_objects(0.10)
        elif kind == "aws_small":
            self._aws(self.aev.batch(self.s.model.actual))
        elif kind == "aws_large":
            self.large_aws(0.02)
        elif kind == "zones":
            self._zones(*self.zev.batch(self.s.model.actual["zones"]))
        else:
            getattr(self, kind)()

    # ------------------------------------------------------------------ queries
    def keysets(self, k):
        """One row, about 1 % and 10 % of the rows and (every third step) every row, each with deleted keys: dropped objects,
        keys this run deleted and keys that match nothing."""
        n = len(self.s.om.objects)
        rng = self.rng
        dk = sorted(self.gone) + [x for x in self.dropped if x not in self.s.om.rows]
        dk = rng.sample(dk, min(len(dk), 300)) + scalemodels.ABSENT_KEYS
        ks = [("one", [rng.randrange(n)], dk), ("1pct", rng.sample(range(n), max(1, n // 100)), dk),
              ("10pct", rng.sample(range(n), max(1, n // 10)), dk)]
        return ks + [("all", list(range(n)), dk)] if k % 3 == 0 else ks

    def full(self, want):
        got = self.e.diff()
        mode = self.e.counters()["launch_mode"]
        if self.check:
            if want["full"] is None:
                want["full"] = self.oracle.diff(want["snap"], "default", mode=1, threads=THREADS)
                assert_same_full(got, want["full"], self.s.om.slab, want["snap"].arrays["o.slab"])
                want["got"] = got
            else:
                assert got.diff(want["got"]) == [], got.describe_first_mismatch(want["got"])  # the same tables: the same answer
        self.results.append(got)
        self.seen["full"] += 1
        return mode

    def keys(self, want, ks):
        for what, rows, dk in ks:
            got = self.e.diff_keys(rows, dk)
            if self.check:
                ref = self.oracle.diff_keys(want["snap"], rows, dk, mode=1)
                assert got.diff(ref) == [], (what, got.describe_first_mismatch(ref))
            want.setdefault("keys", {})[what] = got
        self.seen["keys"] += 1

    def read_set(self, want, ks):
        for what, rows, dk in ks:
            got = read_set_got(self.e, rows, dk)
            if self.check:
                ref = readset_ref.read_set(self.s.om.objects, self.s.model.actual, "default", rows, dk)
                assert got == ref, (what, {k: (len(got[k]), len(ref[k])) for k in got})
            want.setdefault("read_set", {})[what] = got
        self.seen["read_set"] += 1

    def bindings(self, want):
        got = self.e.bindings_diff(self.b).ops.tolist()
        if self.check:
            assert got == self.oracle.bindings_diff(want["snap"], self.b).ops.tolist()
        self.seen["bindings"] += 1
        return got

    def device(self, want):
        cs = self.e.diff_device()
        if self.gpu:
            from test_gpu_scale_models import assert_same, device_changeset
            if self.check:
                assert_same(self.g, device_changeset(self.g.abi, cs), want["got"], "diff_device")
        elif self.check:
            assert int(cs.n_ops) == len(want["full"].ops) and list(cs.section_begin) == [int(x) for x in want["full"].section_begin]
        self.seen["device"] += 1

    def export(self, want, step):
        if self.check:
            x = check_export(self.g, self.e, want["snap"], BOTH if step % 2 == 0 else self.rng.choice([OBJ, ACT]))
        else:
            x = self.e.export(BOTH if step % 2 == 0 else self.rng.choice([OBJ, ACT]))
        self.seen["export"] += 1
        return x

    def restore(self, want, ks):
        """The export loaded into the second engine answers the full diff and diff_keys as the main engine does."""
        x = self.e.export(BOTH)
        self.keep.append(x)
        self.e2.load(x)
        if self.check:
            xslab = np.ctypeslib.as_array(x.objects.slab, shape=(max(1, x.objects.slab_len),))[:x.objects.slab_len]
            assert_same_full(self.e2.diff(), want["full"], xslab, want["snap"].arrays["o.slab"])
            for what, rows, dk in ks:
                got = self.e2.diff_keys(rows, dk)
                assert got.diff(want["keys"][what]) == [], (what, got.describe_first_mismatch(want["keys"][what]))
        self.seen["restore"] += 1

    def sufficiency(self, want, ks):
        """After the deltas: the second engine, loaded from the export, gets every AWS row outside the read set of a keyset
        rewritten (test_read_set.rewrite_outside); its diff_keys stays the main engine's."""
        x = self.e.export(BOTH)
        self.keep.append(x)
        self.e2.load(x)
        for what, rows, dk in ks[1:3]:
            rs = want["read_set"][what]
            apply_rows(self.g, self.e2, self.s.model.actual, rewrite_outside(self.s.model.actual, rs, dk, random.Random(len(rows))))
            if self.check:
                got = self.e2.diff_keys(rows, dk)
                assert got.diff(want["keys"][what]) == [], (what, got.describe_first_mismatch(want["keys"][what]))
            self.e2.load(x)
        self.seen["sufficiency"] += 1

    def settle(self, want, first):
        """Full diffs after the queries that followed a mutation: until one is replayed, at most six in all (GPU; the first full
        diff after the mutation was eager), or as many as the GPU run needed (schedule), or none (host simulation)."""
        if self.schedule is not None:
            modes = [first] + [self.full(want) for _ in range(self.schedule.pop(0))]
        elif self.gpu:
            modes = [first]
            while modes[-1] != 2:
                assert len(modes) < 6, modes
                modes.append(self.full(want))
            assert modes[0] == 0 and set(modes[1:-1]) <= {0, 1}, modes  # (gar_diff_device among the queries may have recorded)
        else:
            modes = [first]
        self.counts.append(len(modes) - 1)
        self.modes.append(modes)
        return modes

    # ------------------------------------------------------------------ one step
    def step(self, k, kinds):
        for kind in kinds:
            self.mutate(kind)
        want = {"snap": self.g.pack(self.s.om.objects, self.s.model.actual) if self.check else None, "full": None}
        self.keep.append(want["snap"])
        first = self.full(want)
        if self.gpu:
            assert first == 0, (kinds, first)  # the recording of the old tables is never replayed
        ks = self.keysets(k)
        self.keys(want, ks)
        self.read_set(want, ks)
        bops = self.bindings(want)
        if self.gpu:  # (the host simulation's device result is a second full diff: checked once per few steps below)
            self.device(want)
        self.export(want, k)
        if k % 3 == 2:
            self.restore(want, ks)
        if k % 4 == 3:
            self.sufficiency(want, ks)
        modes = self.settle(want, first)
        # each query again on the settled snapshot (its buffers fit): the same answer, and the next full diff replays if the
        # last one did
        small, qs = ks[:2], ("keys", "bindings", "device", "read_set", "export")
        for q in qs if self.gpu else qs[k % len(qs):][:1]:
            if q == "keys":
                for what, rows, dk in small:
                    got = self.e.diff_keys(rows, dk)
                    assert not self.check or got.diff(want["keys"][what]) == []
            elif q == "read_set":
                for what, rows, dk in small:
                    assert not self.check or read_set_got(self.e, rows, dk) == want["read_set"][what]
            elif q == "bindings":
                assert self.e.bindings_diff(self.b).ops.tolist() == bops or not self.check
            elif q == "device":
                self.device(want)
            else:
                self.e.export(BOTH)
            mode = self.full(want)
            if self.schedule is None and self.gpu and modes[-1] == 2:
                assert mode == 2, (q, mode)

    def run(self, n_steps):
        """n_steps steps: every mutation kind at least once (in a seeded order), each step now and then preceded by a small
        object or AWS delta with no diff in between (a worker applies several deltas, then diffs).  Zone deltas and compactions
        always are: what the next prepare rebuilds after them must include what the delta before them changed."""
        plan = list(MUTATIONS) + [self.rng.choice(MUTATIONS) for _ in range(max(0, n_steps - len(MUTATIONS)))]
        self.rng.shuffle(plan)
        for k, kind in enumerate(plan[:max(n_steps, len(MUTATIONS))]):
            kinds = [kind]
            if kind in ("zones", "compact") or self.rng.random() < 0.4:
                kinds.insert(0, self.rng.choice(["obj_small", "aws_small"]))
            self.step(k, kinds)
        return self

    def assert_coverage(self, tiles):
        for kind in MUTATIONS + QUERIES:
            assert self.seen[kind] > 0, kind
        if tiles:
            small = {lv: self.spliced[lv] for lv in LEVELS if self.spliced[lv] <= 4 * TILE}
            assert not small, small


def lifecycle(garecon, oracle, engine, second, name, seed, n, n_steps, gpu, **kw):
    return Lifecycle(garecon, oracle, engine, second, name, seed, n, gpu, **kw).run(n_steps)


# ------------------------------------------------------------------ host simulation

@pytest.fixture(scope="module")
def hostlib(garecon):
    import __graft_entry__ as ge
    return garecon.abi.load_library(ge.build_hostsim())


@pytest.mark.parametrize("name,seed", [("rand", 0), ("rand", 1), ("bindings", 2)])
def test_hostsim_lifecycle(garecon, oracle, hostlib, name, seed):
    with garecon.Engine(cluster_name="default", lib=hostlib) as e, garecon.Engine(cluster_name="default", lib=hostlib) as e2:
        lc = lifecycle(garecon, oracle, e, e2, name, seed, 800, len(MUTATIONS), gpu=False)
    lc.assert_coverage(tiles=False)


# ------------------------------------------------------------------ GPU

GPU_RUNS = [(name, seed, 20_000) for name in ("rand", "hot", "multilbi", "bindings") for seed in (0, 1)] + [("rand", 2, 60_000)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,seed,n", GPU_RUNS)
def test_gpu_lifecycle(garecon, oracle, monkeypatch, name, seed, n):
    with _engine(garecon, monkeypatch, False) as e, garecon.Engine(cluster_name="default") as e2:
        lc = lifecycle(garecon, oracle, e, e2, name, seed, n, 12, gpu=True)
    lc.assert_coverage(tiles=True)
    print(f"{name} seed {seed} n {n}: spliced rows {dict(lc.spliced)}, scan tiles "
          f"{ {lv: -(-lc.spliced[lv] // TILE) for lv in LEVELS} }, full diffs per step {lc.counts}")
    if seed == 0:  # the control: never recorded, the same full diffs on the same schedule
        with _engine(garecon, monkeypatch, True) as e, garecon.Engine(cluster_name="default") as e2:
            ctl = lifecycle(garecon, oracle, e, e2, name, seed, n, 12, gpu=True, check=False, schedule=lc.counts)
        assert {m for modes in ctl.modes for m in modes} == {0}
        _same_results(lc, ctl)
