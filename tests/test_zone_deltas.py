"""Zone deltas (gar_snapshot_apply_zones): hosted zones added (with their record sets) and removed on the resident AWS tables.
After every delta the engine must answer exactly as a fresh gar_snapshot_load of the AWS model the tests hold, against the
oracle: full diff, incremental diff and the EndpointGroupBinding set-diff (and, on the GPU, the device-resident result byte
for byte).  Zone deltas interleave with object deltas and AWS deltas; a deltas.ActualMirror runs in lockstep, so every result
tuple and the AWS slab after a compaction are checked too.  Zone order matters: the zone walk takes the first row whose name
matches, so the hand-built cases check subzones, duplicate names, deleted zones with orphans and re-added owned records."""
import copy
import ctypes
import importlib
import random
import subprocess
import tempfile
import textwrap
from pathlib import Path

import numpy as np
import pytest

import egbcases
import randmodel
from test_actual_deltas import AwsEvents, AwsModel, apply_delta, check_all, deltas_mod
from test_launch_replay import Sequence, _engine, _same_results
from test_object_deltas import Events, Mirror, assert_same_full

REPO = Path(__file__).resolve().parent.parent
NONE = 0xFFFFFFFF
R53_CREATE, R53_UPSERT_A, R53_DELETE_RECORD = 8, 9, 10
D_NO_HOSTED_ZONE = 9


def _act(garecon, struct):
    return garecon.tables.columns(struct, garecon.tables.ACT_TABLES)


class State:
    """An engine with its mirrors: objects (Mirror), AWS tables as dicts (AwsModel: what the oracle is given) and as columns
    laid out like the resident tables (deltas.ActualMirror: result tuples and the slab)."""

    def __init__(self, garecon, oracle, engine, objects, actual, oracle_mode=0):
        self.g, self.oracle, self.e, self.mode = garecon, oracle, engine, oracle_mode
        self.snap = garecon.pack(objects, actual)
        engine.load(self.snap)
        self.om, self.model = Mirror(objects, self.snap), AwsModel(actual, self.snap)
        self.am = deltas_mod().ActualMirror(_act(garecon, self.snap.actual))

    def msnap(self):
        return self.g.pack(self.om.objects, self.model.actual)

    def aws(self, d):
        """An AWS delta (AwsModel.apply's form) on the engine and both mirrors."""
        res = apply_delta(self.g, self.e, self.model, d)
        rows = _act(self.g, d["_rows"].actual) if d["_rows"] is not None else None
        want = self.am.apply(rows, [t for t, _ in d.get("lbs", [])], [t for t, _ in d.get("accs", [])], [z for z, _ in d.get("zones", [])],
                             d.get("lb_deleted", []), d.get("acc_deleted", []))
        assert tuple(res) == tuple(want[k] for k in self.g.abi.ActualDeltaResult.FIELDS)
        return res

    def zones(self, added=(), deleted=()):
        """added: [(added_at, zone dict)] with added_at non-decreasing; deleted: resident zone rows.  Applies the zone delta to
        the engine and both mirrors; checks the result against both.  -> (result, new row of each added zone)."""
        added = list(added)
        packed = self.g.pack([], {"zones": [z for _, z in added]}) if added else None
        at = [a for a, _ in added]
        res = self.e.apply_zones(packed.actual if packed else None, at, list(deleted))
        want = self.am.apply_zones(_act(self.g, packed.actual) if packed else None, at, list(deleted))
        assert tuple(res) == tuple(want[k] for k in self.g.abi.ZoneDeltaResult.FIELDS), (tuple(res), want)
        # the header's rule on the dict model
        old, gone = self.model.actual["zones"], set(deleted)
        new, k = [], 0
        for r in range(len(old) + 1):
            while k < len(added) and added[k][0] == r:
                new.append(added[k][1])
                k += 1
            if r < len(old) and r not in gone:
                new.append(old[r])
        self.model.actual["zones"] = new
        base = 0
        if added:
            base = (self.model.slab_len + 15) & ~15
            self.model.slab_len = base + int(packed.actual.slab_len)
        recs = [r for z in new for r in z.get("records", [])]
        assert tuple(res) == (len(new), len(recs), sum(len(r.get("values", [])) for r in recs), base, self.model.slab_len)
        return res, [a - sum(1 for d in deleted if d < a) + i for i, a in enumerate(at)]

    def check(self, rows=(), deleted_keys=(), bindings=None):
        msnap = self.msnap()
        got = self.e.diff()
        assert_same_full(got, self.oracle.diff(msnap, "default", mode=1), self.om.slab, msnap.arrays["o.slab"])
        if rows or deleted_keys:
            got_k = self.e.diff_keys(list(rows), list(deleted_keys))
            want_k = self.oracle.diff_keys(msnap, list(rows), list(deleted_keys), mode=self.mode)
            assert got_k.diff(want_k) == [], got_k.describe_first_mismatch(want_k)
        if bindings is not None:
            assert self.e.bindings_diff(bindings).ops.tolist() == self.oracle.bindings_diff(msnap, bindings).ops.tolist()
        return got


class ZoneEvents:
    """Random changes of the zone set over a randmodel AWS model: adds at the front, in the middle and at the end (empty,
    with records, subzones named after a record name, duplicates of a resident name), deletes, a deleted zone re-added under
    the same name elsewhere, and now and then every zone deleted."""

    def __init__(self, seed):
        self.rng = random.Random(seed * 977 + 3)
        self.pool = randmodel.make(seed + 9000, n_objects=30)[1].get("zones", [])
        self.serial = 0

    def _new_zone(self, zones):
        rng = self.rng
        src = rng.choice(zones + self.pool)
        c = rng.random()
        self.serial += 1
        if c < 0.25:
            return {"id": f"/hostedzone/N{self.serial}", "name": src["name"], "records": []}
        if c < 0.5:
            return dict(copy.deepcopy(src), id=f"/hostedzone/N{self.serial}")
        if c < 0.75 and src.get("records"):
            name = rng.choice(src["records"])["name"]
            return {"id": f"/hostedzone/N{self.serial}", "name": name, "records": [copy.deepcopy(r) for r in src["records"] if r["name"] == name]}
        recs = copy.deepcopy(src.get("records", [])[:rng.randrange(0, 4)])
        return {"id": f"/hostedzone/N{self.serial}", "name": f"zn{self.serial}.example.net.", "records": recs}

    def batch(self, zones):
        rng, n = self.rng, len(zones)
        if n and rng.random() < 0.08:
            return [], list(range(n))
        deleted = rng.sample(range(n), rng.randrange(0, min(n, 3) + 1))
        added = []
        if deleted and rng.random() < 0.4:  # deleted, and listed again under the same name elsewhere
            added.append((rng.randrange(n + 1), copy.deepcopy(zones[deleted[0]])))
        for _ in range(rng.randrange(0, 4)):
            added.append((rng.choice([0, n, rng.randrange(n + 1)]), self._new_zone(zones)))
        added.sort(key=lambda x: x[0])
        return added, deleted


def run_sequence(garecon, oracle, engine, seed, n_objects, n_batches, oracle_mode, device=False):
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=n_objects, n_bindings=3 * n_objects)
    b = garecon.pack_bindings(bindings, known)
    s = State(garecon, oracle, engine, objects, actual, oracle_mode)
    oevents, aevents, zevents = Events(seed, actual), AwsEvents(seed), ZoneEvents(seed)
    rng = random.Random(seed)
    s.e.diff()  # the deltas below must drop a prepared snapshot
    for _ in range(n_batches):
        c = rng.random()
        if c < 0.3:
            upserts, deleted = oevents.batch(s.om.objects)
            usnap = garecon.pack(upserts, None) if upserts else None
            engine.apply_objects(usnap.objects if usnap else None, deleted)
            s.om.apply(upserts, deleted, usnap)
        elif c < 0.5:
            s.aws(aevents.batch(s.model.actual))
        s.zones(*zevents.batch(s.model.actual["zones"]))
        rows = rng.sample(range(len(s.om.objects)), min(len(s.om.objects), 8))
        check_all(garecon, oracle, engine, s.om, s.model, b, rows, [], oracle_mode)
        if device:
            from test_gpu_scale_models import assert_same, device_changeset
            assert_same(garecon, device_changeset(garecon.abi, engine.diff_device()), engine.diff(), "diff_device")
    # compaction after zone deltas: the AWS slab is deltas.compact_actual of the mirror, byte for byte; answers unchanged
    before = engine.diff()
    res = engine.compact(garecon.abi.COMPACT_ACTUAL)
    assert res.act_slab_len == s.am.compact()
    got = engine.read_slab(garecon.abi.COMPACT_ACTUAL, 0, res.act_slab_len)
    assert np.array_equal(got, np.asarray(s.am.cur["slab"], dtype=np.uint8))
    assert engine.diff().diff(before) == []
    check_all(garecon, oracle, engine, s.om, s.model, b, list(range(0, len(s.om.objects), 3)), [], oracle_mode)
    return s


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


@pytest.mark.parametrize("seed", range(20))
def test_hostsim_random_sequences(garecon, oracle, hostsim, seed):
    run_sequence(garecon, oracle, hostsim, seed, n_objects=30, n_batches=random.Random(seed).randrange(4, 9), oracle_mode=0)


def test_hostsim_sequence_with_tiny_capacities(garecon, oracle, hostsim, monkeypatch):
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    run_sequence(garecon, oracle, hostsim, 107, n_objects=30, n_batches=6, oracle_mode=0)


# ------------------------------------------------------------------ hand-built zone-walk cases

def _r53(cs):
    """(op code, obj, sub, zone row) of every Route53 op of the object sections, and the orphan deletes (section 3)."""
    sb = [int(x) for x in cs.section_begin]
    own = [(int(o["head"]) & 0xFF, int(o["obj"]), int(o["sub"]), int(o["a0"])) for o in cs.ops[sb[2]:sb[3]]]
    orphans = [(int(o["head"]) & 0xFF, int(o["a0"])) for o in cs.ops[sb[3]:sb[4]]]
    return own, orphans


def _hosted(oracle, garecon, seed=5, n_objects=40):
    """A randmodel cluster and an object row whose R53 ops name a zone for a non-wildcard hostname: (objects, actual, obj, zone
    row, hostname)."""
    objects, actual = randmodel.make(seed, n_objects=n_objects)
    cs = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    own, _ = _r53(cs)
    for code, obj, sub, zone in own:
        if code in (R53_CREATE, R53_UPSERT_A):
            hosts = [h.strip() for h in objects[obj]["annotations"][randmodel.ANN + "route53-hostname"].split(",")]
            h = hosts[sub & 0xFFFFF]
            if not h.startswith("*"):
                return objects, actual, obj, zone, h
    raise AssertionError("no object with Route53 ops in this model")


def _zones_of(own, obj):
    return {z for code, o, _, z in own if o == obj and code in (R53_CREATE, R53_UPSERT_A)}


def walk_cases(garecon, oracle, engine):
    objects, actual, obj, z, host = _hosted(oracle, garecon)
    s = State(garecon, oracle, engine, objects, actual)
    first = s.check()
    # a subzone named after the hostname, listed first: the hostname now names it; deleted again: back to the parent zone
    s.zones([(0, {"id": "/hostedzone/SUB", "name": host + ".", "records": []})])
    own, _ = _r53(s.check())
    assert _zones_of(own, obj) == {0}
    s.zones(deleted=[0])
    assert s.check().diff(first) == []
    # duplicate names: a zone in front of z wins, one behind every zone loses, deleting the front one lets z win again
    name = actual["zones"][z]["name"]
    _, (front,) = s.zones([(z, {"id": "/hostedzone/DUP1", "name": name, "records": []})])
    assert front == z
    own, _ = _r53(s.check())
    assert _zones_of(own, obj) == {z}
    n = len(s.model.actual["zones"])
    assert all(code == R53_CREATE for code, o, _, zz in own if o == obj and zz == z)  # the empty duplicate has no record yet
    _, (behind,) = s.zones([(n, {"id": "/hostedzone/DUP2", "name": name, "records": copy.deepcopy(actual["zones"][z]["records"])})])
    assert behind == n
    own2, _ = _r53(s.check())
    assert own2 == own
    s.zones(deleted=[z])  # the one in front: the resident zone wins again
    own3, _ = _r53(s.check())
    assert _zones_of(own3, obj) == {z}
    s.zones(deleted=[z])  # the resident zone: the copy behind every other zone wins, with the same record sets
    own4, _ = _r53(s.check())
    assert _zones_of(own4, obj) == {len(s.model.actual["zones"]) - 1}
    assert [c for c, o, _, _ in own4 if o == obj] == [c for c, o, _, _ in _r53(first)[0] if o == obj]


def orphan_cases(garecon, oracle, engine):
    objects, actual = randmodel.make(5, n_objects=40)
    s = State(garecon, oracle, engine, objects, actual)
    first = s.check()
    own, orphans = _r53(first)
    zs = sorted({zz for _, zz in orphans})
    assert zs, "the model has orphan record sets"
    z = zs[0]
    s.zones(deleted=[z])
    own2, orphans2 = _r53(s.check())
    assert len(orphans2) == len(orphans) - sum(1 for _, zz in orphans if zz == z)
    # every zone that could hold an object's hostname deleted: that object reports GAR_D_NO_HOSTED_ZONE
    objects, actual, obj, z, host = _hosted(oracle, garecon)
    s = State(garecon, oracle, engine, objects, actual)
    s.check()
    labels = host.split(".")
    suffixes = {".".join(labels[i:]) + "." for i in range(len(labels))}
    gone = [r for r, x in enumerate(actual["zones"]) if x["name"] in suffixes]
    s.zones(deleted=gone)
    cs = s.check()
    assert (int(cs.status_r53[obj]) >> 8) & 0xFF == D_NO_HOSTED_ZONE


def owned_records_cases(garecon, oracle, engine):
    """A zone holding records an object owns (A, TXT, and \\052 wildcard names) is deleted and added back: the object's
    creates become the upserts / no-ops of the first snapshot again."""
    for seed in range(5, 60):
        objects, actual = randmodel.make(seed, n_objects=40)
        zs = [r for r, x in enumerate(actual["zones"]) if any(rec["name"].startswith("\\052") for rec in x.get("records", []))]
        if zs:
            break
    else:
        raise AssertionError("no model with wildcard records")
    z = zs[0]
    s = State(garecon, oracle, engine, objects, actual)
    first = s.check()
    own, _ = _r53(first)
    assert any(zz == z for code, _, _, zz in own if code in (R53_CREATE, R53_UPSERT_A)) or any(zz == z for _, zz in _r53(first)[1])
    zone = copy.deepcopy(actual["zones"][z])
    s.zones(deleted=[z])
    s.check()
    s.zones([(z, zone)])
    assert s.check().diff(first) == []


def row_formula_case(garecon, oracle, engine):
    """The header's row formulas address the zones after a delta: a later gar_snapshot_apply_actual replaces the record list of
    a surviving zone and of a new zone at the rows the formulas give (the AWS delta checks the names at those rows)."""
    objects, actual = randmodel.make(9, n_objects=30)
    for i, x in enumerate(actual["zones"]):
        x["name"] = f"u{i}.{x['name']}"  # unique names: a wrong row fails the AWS delta's name check
    s = State(garecon, oracle, engine, objects, actual)
    s.check()
    n = len(actual["zones"])
    deleted = [0, n // 2]
    added = [(1, {"id": "/hostedzone/F1", "name": "f1.example.org.", "records": []}),
             (n, {"id": "/hostedzone/F2", "name": "f2.example.org.", "records": copy.deepcopy(actual["zones"][1].get("records", []))})]
    _, rows = s.zones(added, deleted)
    r = n - 1  # a surviving resident row
    new_r = r - sum(1 for d in deleted if d < r) + sum(1 for a, _ in added if a <= r)
    assert s.model.actual["zones"][new_r]["name"] == actual["zones"][r]["name"]
    recs = copy.deepcopy(actual["zones"][2].get("records", []))[:3]
    s.aws({"zones": [(new_r, recs), (rows[1], [])]})
    assert s.model.actual["zones"][rows[1]]["name"] == "f2.example.org."
    s.check(rows=range(0, len(objects), 2))


def full_relist_case(garecon, oracle, engine, fresh):
    """A full AWS re-list as deltas: every load balancer, accelerator and zone deleted, then a mutated model added back.  The
    engine answers as a load of that model (oracle and a fresh engine)."""
    objects, actual = randmodel.make(13, n_objects=40)
    s = State(garecon, oracle, engine, objects, actual)
    s.check()
    _, mutated = randmodel.make(14, n_objects=40)
    mutated["zones"] = mutated.get("zones", []) + copy.deepcopy(actual["zones"][:2])
    s.aws({"lb_deleted": list(range(len(actual["lbs"]))), "acc_deleted": list(range(len(actual["accelerators"]))),
           "lbs": [(NONE, x) for x in mutated.get("lbs", [])], "accs": [(NONE, x) for x in mutated.get("accelerators", [])]})
    s.zones([(0, x) for x in mutated["zones"]], list(range(len(actual["zones"]))))
    assert s.model.actual["lbs"] == mutated.get("lbs", []) and s.model.actual["zones"] == mutated["zones"]
    got = s.check(rows=range(0, len(objects), 3))
    msnap = garecon.pack(objects, mutated)
    fresh.load(msnap)
    want = fresh.diff()
    assert_same_full(got, want, s.om.slab, msnap.arrays["o.slab"])


def test_hostsim_subzones_and_duplicate_names(garecon, oracle, hostsim):
    walk_cases(garecon, oracle, hostsim)


def test_hostsim_deleted_zones_drop_their_orphans(garecon, oracle, hostsim):
    orphan_cases(garecon, oracle, hostsim)


def test_hostsim_readded_zone_with_owned_records(garecon, oracle, hostsim):
    owned_records_cases(garecon, oracle, hostsim)


def test_hostsim_row_formulas_address_later_aws_deltas(garecon, oracle, hostsim):
    row_formula_case(garecon, oracle, hostsim)


def test_hostsim_full_relist_as_deltas(garecon, oracle, hostsim):
    import __graft_entry__ as ge
    with garecon.Engine(cluster_name="default", lib=garecon.abi.load_library(ge.build_hostsim())) as fresh:
        full_relist_case(garecon, oracle, hostsim, fresh)


# ------------------------------------------------------------------ refused deltas change nothing

BREAKAGES = ["deleted_range", "deleted_twice", "at_range", "at_decreasing", "lb_rows", "acc_rows", "null_at", "null_deleted", "csr",
             "string", "enum"]


def refused_cases(garecon, engine, breakage):
    abi = garecon.abi
    objects, actual = randmodel.make(5, n_objects=20)
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    before = engine.diff()
    n = len(actual["zones"])
    z = copy.deepcopy(actual["zones"][0])
    packed = garecon.pack([], {"zones": [z, z]})
    args = dict(added_at=[0, 1], deleted=[1])
    if breakage == "deleted_range":
        args["deleted"] = [n]
    elif breakage == "deleted_twice":
        args["deleted"] = [2, 2]
    elif breakage == "at_range":
        args["added_at"] = [0, n + 1]
    elif breakage == "at_decreasing":
        args["added_at"] = [2, 1]
    elif breakage == "lb_rows":
        packed = garecon.pack([], {"zones": [z, z], "lbs": actual["lbs"][:1]})
    elif breakage == "acc_rows":
        packed = garecon.pack([], {"zones": [z, z], "accelerators": actual["accelerators"][:1]})
    elif breakage == "csr":
        packed.arrays["zone_rec_begin"][1] = packed.arrays["zone_rec_begin"][2] + 1
    elif breakage == "string":
        packed.arrays["zone_name"][1] = (4 << 40) | int(packed.actual.slab_len)
    elif breakage == "enum":
        packed.arrays["rec_type"][0] = 9
    if breakage.startswith("null"):
        ok = np.zeros(2, dtype=np.uint32)
        d = abi.GarZoneDelta(ctypes.pointer(packed.actual), None if breakage == "null_at" else ok.ctypes.data_as(abi._u32p), 1,
                             ok.ctypes.data_as(abi._u32p) if breakage == "null_at" else None)
        rc = engine.lib.gar_snapshot_apply_zones(engine._h, ctypes.byref(d), ctypes.byref(abi.GarZoneDeltaResult()))
        assert rc == abi.GAR_E_INVALID
    else:
        with pytest.raises(garecon.GarError) as ei:
            engine.apply_zones(packed.actual, **args)
        assert ei.value.rc == abi.GAR_E_INVALID
    assert engine.diff().diff(before) == []
    assert tuple(engine.apply_zones()) == (n, int(snap.actual.n_records), int(snap.actual.n_values), 0, int(snap.actual.slab_len))
    assert engine.diff().diff(before) == []


@pytest.mark.parametrize("breakage", BREAKAGES)
def test_hostsim_invalid_zone_delta_changes_nothing(garecon, hostsim, breakage):
    refused_cases(garecon, hostsim, breakage)


def test_hostsim_zone_delta_before_load_is_a_state_error(garecon):
    import __graft_entry__ as ge
    with garecon.Engine(cluster_name="default", lib=garecon.abi.load_library(ge.build_hostsim())) as e:
        with pytest.raises(garecon.GarError) as ei:
            e.apply_zones(deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE


def test_ctypes_zone_delta_struct_sizes_match_header(garecon):
    src = textwrap.dedent('''
        #include <stdio.h>
        #include "garecon.h"
        int main(void) { printf("%zu %zu\\n", sizeof(gar_zone_delta), sizeof(gar_zone_delta_result)); return 0; }
    ''')
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(REPO / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout.split()
    abi = garecon.abi
    assert [int(x) for x in out] == [ctypes.sizeof(abi.GarZoneDelta), ctypes.sizeof(abi.GarZoneDeltaResult)]


# ------------------------------------------------------------------ recorded launches after a zone delta

class ZoneSequence(Sequence):
    """tests/test_launch_replay.py's sequence with one more mutation: a zone delta."""

    def __init__(self, *a, **kw):
        self.zev = ZoneEvents(7)
        super().__init__(*a, **kw)

    def _load(self, objects, actual):
        super()._load(objects, actual)
        self.st = State.__new__(State)
        self.st.g, self.st.e, self.st.model = self.g, self.e, self.model
        self.st.am = deltas_mod().ActualMirror(_act(self.g, self.snap.actual))

    def zones(self):
        self.st.zones(*self.zev.batch(self.model.actual["zones"]))


def replay_ops(seq):
    seq.warm()
    seq.settle("load")
    for op in ("zones", "diff", "zones", "zones", "objects", "zones"):
        seq.run(op)
        seq.warm()
        seq.settle(op + "+warm")
    return seq


def test_hostsim_zone_delta_replay_bookkeeping(garecon, oracle, hostsim):
    seq = replay_ops(ZoneSequence(garecon, oracle, hostsim, 4, 60, 0, gpu=False))
    assert {m for ms in seq.after.values() for modes in ms for m in modes} == {0}


# ------------------------------------------------------------------ table-level churn (deltas.zone_churn: what profiles/zone_delta_bench.py runs)

def zone_churn_sequence(garecon, engine, snap, seed, n_batches=3):
    """Load `snap`; apply zone_churn batches (adds with records, a subzone, a duplicate in front, deletes) interleaved with an
    aws_churn batch; check every result against deltas.ActualMirror.  -> (mirror, mirror snapshot)."""
    deltas, tables = deltas_mod(), garecon.tables
    engine.load(snap)
    engine.diff_raw()
    m = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    rng = np.random.default_rng(seed)
    for i in range(n_batches):
        d = deltas.zone_churn(m, rng, n_add=10, rec_frac=0.01, n_del=3 * (i % 2), serial=i)
        keep, added = deltas.actual_struct(d["added"])
        res = engine.apply_zones(added, d["added_at"], d["deleted"])
        want = m.apply_zones(**d)
        assert tuple(res) == tuple(want[k] for k in garecon.abi.ZoneDeltaResult.FIELDS)
        if i == 0:
            a = deltas.aws_churn(m, rng)
            keep, rows = deltas.actual_struct(a["rows"])
            res = engine.apply_actual(rows, a["lb_target"], a["acc_target"], a["zone_target"], a["lb_deleted"], a["acc_deleted"])
            want = m.apply(**a)
            assert tuple(res) == tuple(want[k] for k in garecon.abi.ActualDeltaResult.FIELDS)
    return m, m.snapshot(tables.columns(snap.objects, tables.OBJ_TABLES))


def test_hostsim_zone_churn_matches_actual_mirror(garecon, oracle, hostsim):
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, 3000)
    m, msnap = zone_churn_sequence(garecon, hostsim, snap, 23)
    got = hostsim.diff()
    want = oracle.diff(msnap, snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    rows = list(range(0, int(msnap.objects.n_objects), 97))
    got = hostsim.diff_keys(rows)
    want = oracle.diff_keys(msnap, rows, [], cluster=snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


# ------------------------------------------------------------------ GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(600, 612))
def test_gpu_random_sequences(garecon, oracle, engine, seed):
    run_sequence(garecon, oracle, engine, seed, n_objects=80, n_batches=random.Random(seed).randrange(4, 9), oracle_mode=1, device=True)


@pytest.mark.gpu
def test_gpu_zone_walk_cases(garecon, oracle, engine):
    walk_cases(garecon, oracle, engine)
    orphan_cases(garecon, oracle, engine)
    owned_records_cases(garecon, oracle, engine)
    row_formula_case(garecon, oracle, engine)
    with garecon.Engine(cluster_name="default") as fresh:
        full_relist_case(garecon, oracle, engine, fresh)


@pytest.mark.gpu
def test_gpu_invalid_and_state_errors(garecon, engine):
    for breakage in BREAKAGES:
        refused_cases(garecon, engine, breakage)
    with garecon.Engine(cluster_name="default") as e:
        with pytest.raises(garecon.GarError) as ei:
            e.apply_zones(deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE


@pytest.mark.gpu
def test_gpu_attached_and_sharded_are_state_errors(garecon):
    import torch
    objects, actual = randmodel.make(5, n_objects=20)
    snap = garecon.pack(objects, actual)
    tables = garecon.tables
    keep = []

    def dev(struct, tabs):
        s = type(struct)()
        ctypes.pointer(s)[0] = struct
        for t, (nf, cl) in tabs.items():
            for name, kind in cl:
                arr = tables.columns(struct, {t: (nf, [(name, kind)])})[name]
                x = torch.from_numpy(np.ascontiguousarray(arr).copy() if arr.size else np.zeros(1, dtype=arr.dtype)).cuda()
                keep.append(x)
                setattr(s, name, ctypes.cast(ctypes.c_void_p(x.data_ptr()), type(getattr(s, name))))
        sl = torch.from_numpy(np.concatenate([tables.columns(struct, {})["slab"], np.zeros(64, dtype=np.uint8)])).cuda()
        keep.append(sl)
        s.slab = ctypes.cast(ctypes.c_void_p(sl.data_ptr()), type(s.slab))
        return s

    with garecon.Engine(cluster_name="default") as e:
        e.attach_device(dev(snap.objects, tables.OBJ_TABLES), dev(snap.actual, tables.ACT_TABLES))
        before = e.diff()
        with pytest.raises(garecon.GarError) as ei:
            e.apply_zones(deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE
        assert e.diff().diff(before) == []
        e.load(snap)
        e.shard_route(garecon.abi.GarShard(0, 1, 0, 0, 0, 0, 0, 0, 0), 1)
        with pytest.raises(garecon.GarError) as ei:
            e.apply_zones(deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE


@pytest.mark.gpu
@pytest.mark.parametrize("no_graph", [False, True])
def test_gpu_replay_after_zone_deltas(garecon, oracle, monkeypatch, no_graph):
    """After a zone delta the recording of the old tables is never replayed: full diffs go eager, record (1), replay (2),
    equal to the oracle throughout; with GAR_NO_GRAPH=1 the same answers, never recorded."""
    with _engine(garecon, monkeypatch, False) as e:
        seq = replay_ops(ZoneSequence(garecon, oracle, e, 4, 80, 1, gpu=True))
    for modes in seq.after["zones"]:
        assert modes[0] == 0 and modes[-2:] == [1, 2], modes
    if no_graph:
        with _engine(garecon, monkeypatch, True) as e:
            ctl = replay_ops(ZoneSequence(garecon, oracle, e, 4, 80, 1, gpu=True, schedule=seq.counts))
        assert {m for ms in ctl.after.values() for modes in ms for m in modes} == {0}
        _same_results(seq, ctl)


@pytest.mark.gpu
def test_gpu_zone_churn_at_scale(garecon, oracle, engine):
    """configs[2] at 10^6 objects with profiles/zone_delta_bench.py's three zone deltas (one empty zone; ten zones holding ~1 %
    of the records, one a subzone of a busy zone and one a duplicate name in front; the ten zones with the most records
    deleted): after each, the full diff equals a fresh load of the mirrored tables; after the last, the oracle too."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    deltas, tables = deltas_mod(), garecon.tables
    snap = synth.generate(3, 1_000_000)
    engine.load(snap)
    engine.diff_raw()
    m = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    o_cols = tables.columns(snap.objects, tables.OBJ_TABLES)
    rng = np.random.default_rng(2)
    arms = [lambda: deltas.zone_churn(m, rng, n_add=1, rec_frac=0.0, serial=0), lambda: deltas.zone_churn(m, rng, n_add=10, rec_frac=0.01, serial=1),
            lambda: deltas.largest_zones_deleted(m, 10)]
    with garecon.Engine(cluster_name=snap.cluster) as fresh:
        for arm in arms:
            d = arm()
            keep, added = deltas.actual_struct(d["added"]) if d["added"] is not None else (None, None)
            res = engine.apply_zones(added, d["added_at"], d["deleted"])
            want = m.apply_zones(**d)
            assert tuple(res) == tuple(want[k] for k in garecon.abi.ZoneDeltaResult.FIELDS)
            got = engine.diff()
            msnap = m.snapshot(o_cols)
            fresh.load(msnap)
            ref = fresh.diff()
            assert got.diff(ref) == [], got.describe_first_mismatch(ref)
    want = oracle.diff(msnap, snap.cluster, mode=1, threads=8)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
