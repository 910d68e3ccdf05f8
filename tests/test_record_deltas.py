"""Record deltas (gar_snapshot_apply_records) and the record read set (gar_read_records).

After every record delta the engine must answer exactly as a fresh gar_snapshot_load of the AWS model the tests hold, against
the oracle (full diff, incremental diff, EndpointGroupBinding set-diff), and its exported AWS tables must equal the compacted
layout of a deltas.ActualMirror run in lockstep.  Record deltas interleave with object, AWS and zone deltas and compactions.
The record read set is checked against a Python restatement of its rule, for sufficiency (every record outside it rewritten,
inserted around or deleted leaves gar_diff_keys' answer unchanged up to the renumbering of record and value rows), and in the
worker's refresh loop at record granularity.  The cases run on the host simulation (CPU tier) and on the GPU."""
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
import hotkeys
import multilbi
import randmodel
import scalemodels
import test_read_set as trs
from oracle import pyref
from test_actual_deltas import AwsEvents, check_all, deltas_mod
from test_object_deltas import Events
from test_zone_deltas import State, ZoneEvents, _act

REPO = Path(__file__).resolve().parent.parent
NONE = 0xFFFFFFFF
OBJ, ACT = 1, 2
R53_UPSERT_A, R53_DELETE_RECORD = 9, 10


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


@pytest.fixture(params=["hostsim", pytest.param("gpu", marks=pytest.mark.gpu)])
def eng(request):
    return request.getfixturevalue("hostsim" if request.param == "hostsim" else "engine")


def zone_begins(zones):
    return np.concatenate([[0], np.cumsum([len(z.get("records", [])) for z in zones])]).astype(np.int64)


def splice_model(zones, inserts, deleted):
    """The header's rule on the dict model: inserts = {zone row: [(position inside the zone, record)]}, deleted = global rows."""
    zb, gone, out = zone_begins(zones), set(int(d) for d in deleted), []
    for z, zone in enumerate(zones):
        recs, ins, new, k = zone.get("records", []), inserts.get(z, []), [], 0
        for p in range(len(recs) + 1):
            while k < len(ins) and ins[k][0] == p:
                new.append(ins[k][1])
                k += 1
            if p < len(recs) and zb[z] + p not in gone:
                new.append(recs[p])
        out.append(dict(zone, records=new))
    return out


class RState(State):
    """test_zone_deltas.State with record deltas."""

    def records(self, inserts=(), deleted=()):
        """inserts: [(zone row, [(position inside the zone, record dict)])], zone rows ascending, positions non-decreasing;
        deleted: resident record rows.  Applies the delta to the engine and both mirrors and checks the result against both.
        -> (result, new row of each inserted record)."""
        zones = self.model.actual["zones"]
        zb = zone_begins(zones)
        inserts = [(z, ins) for z, ins in inserts if ins]
        packed = self.g.pack([], {"zones": [dict(zones[z], records=[r for _, r in ins]) for z, ins in inserts]}) if inserts else None
        zt = [z for z, _ in inserts]
        at = [int(zb[z]) + p for z, ins in inserts for p, _ in ins]
        res = self.e.apply_records(packed.actual if packed else None, zt, at, list(deleted))
        want = self.am.apply_records(_act(self.g, packed.actual) if packed else None, zt, at, list(deleted))
        assert tuple(res) == tuple(want[k] for k in self.g.abi.RecordDeltaResult.FIELDS), (tuple(res), want)
        new = splice_model(zones, dict(inserts), deleted)
        self.model.actual["zones"] = new
        base = 0
        if at:
            base = (self.model.slab_len + 15) & ~15
            self.model.slab_len = base + int(packed.actual.slab_len)
        recs = [r for z in new for r in z["records"]]
        assert tuple(res) == (len(recs), sum(len(r.get("values", [])) for r in recs), base, self.model.slab_len)
        dl = sorted(int(d) for d in deleted)
        return res, [a - int(np.searchsorted(dl, a)) + k for k, a in enumerate(at)]

    def check_export(self):
        """The resident AWS tables, exported, equal the mirror's compacted layout column for column."""
        x = self.e.export(ACT)
        got = self.g.tables.columns(x.actual, self.g.tables.ACT_TABLES)
        want = deltas_mod().compact_actual(self.am.cur)
        for k in want:
            assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k


class RecordEvents:
    """Random record-set edits over a dict model: replaced sets (another alias target, other values, another type), inserts at
    a zone's front, end and in between (copies of records from anywhere), deletes, now and then a zone's every record deleted,
    and edits in empty and adjacent empty zones."""

    def __init__(self, seed):
        self.rng = random.Random(seed * 131 + 7)
        self.serial = 0

    def _changed(self, rec, pool):
        r, c = copy.deepcopy(rec), self.rng.random()
        self.serial += 1
        if r.get("alias") is not None and c < 0.5:
            r["alias"] = f"x{self.serial}.awsglobalaccelerator.com."
        elif c < 0.8:
            r["values"] = copy.deepcopy(self.rng.choice(pool).get("values", []))
        else:
            r["type"] = self.rng.choice(["A", "TXT", "CNAME"])
        return r

    def batch(self, zones):
        rng, zb = self.rng, zone_begins(zones)
        pool = [r for z in zones for r in z.get("records", [])]
        if not zones:
            return [], []
        picked = set(rng.sample(range(len(zones)), min(len(zones), rng.randrange(1, 5))))
        empty = [z for z, zone in enumerate(zones) if not zone.get("records")]
        if empty and rng.random() < 0.5:
            picked.update(empty[:2])
        inserts, deleted = [], []
        for z in sorted(picked):
            recs, ins = zones[z].get("records", []), []
            if recs and rng.random() < 0.1:
                deleted += [int(zb[z]) + p for p in range(len(recs))]
            else:
                for p in range(len(recs)):
                    c = rng.random()
                    if c < 0.15:
                        deleted.append(int(zb[z]) + p)
                        ins.append((p, self._changed(recs[p], pool)))
                    elif c < 0.25:
                        deleted.append(int(zb[z]) + p)
                    elif c < 0.35 and pool:
                        ins.append((p, copy.deepcopy(rng.choice(pool))))
            for p in (0, len(recs)):
                if pool and rng.random() < 0.6:
                    ins.append((p, copy.deepcopy(rng.choice(pool))))
            ins.sort(key=lambda x: x[0])
            inserts.append((z, ins))
        return inserts, deleted


def run_sequence(garecon, oracle, engine, seed, n_objects, n_batches, oracle_mode):
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=n_objects, n_bindings=3 * n_objects)
    b = garecon.pack_bindings(bindings, known)
    s = RState(garecon, oracle, engine, objects, actual, oracle_mode)
    oevents, aevents, zevents, revents = Events(seed, actual), AwsEvents(seed), ZoneEvents(seed), RecordEvents(seed)
    rng = random.Random(seed)
    s.e.diff()  # the deltas below must drop a prepared snapshot
    for _ in range(n_batches):
        c = rng.random()
        if c < 0.2:
            upserts, deleted = oevents.batch(s.om.objects)
            usnap = garecon.pack(upserts, None) if upserts else None
            engine.apply_objects(usnap.objects if usnap else None, deleted)
            s.om.apply(upserts, deleted, usnap)
        elif c < 0.35:
            s.aws(aevents.batch(s.model.actual))
        elif c < 0.5:
            s.zones(*zevents.batch(s.model.actual["zones"]))
        elif c < 0.6:
            res = engine.compact(garecon.abi.COMPACT_ACTUAL)
            assert res.act_slab_len == s.am.compact()
            s.model.slab_len = res.act_slab_len
        s.records(*revents.batch(s.model.actual["zones"]))
        rows = rng.sample(range(len(s.om.objects)), min(len(s.om.objects), 8))
        check_all(garecon, oracle, engine, s.om, s.model, b, rows, [], oracle_mode)
        s.check_export()
    return s


@pytest.mark.parametrize("seed", range(16))
def test_hostsim_random_sequences(garecon, oracle, hostsim, seed):
    run_sequence(garecon, oracle, hostsim, seed, n_objects=30, n_batches=random.Random(seed).randrange(4, 9), oracle_mode=0)


def test_hostsim_sequence_with_tiny_capacities(garecon, oracle, hostsim, monkeypatch):
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    run_sequence(garecon, oracle, hostsim, 211, n_objects=30, n_batches=6, oracle_mode=0)


# ------------------------------------------------------------------ the row formulas at the edges

def edge_cases(garecon, oracle, engine):
    objects, actual = randmodel.make(11, n_objects=40)
    zones = actual["zones"]
    pool = [r for z in zones for r in z.get("records", [])]
    # two adjacent empty zones behind a populated one, and an empty zone at the front
    actual["zones"] = [{"id": "/hostedzone/E0", "name": "e0.example.org.", "records": []}] + zones[:2] + [
        {"id": "/hostedzone/E1", "name": "e1.example.org.", "records": []}, {"id": "/hostedzone/E2", "name": "e2.example.org.", "records": []}] + zones[2:]
    s = RState(garecon, oracle, engine, objects, actual)
    s.e.diff()
    zb = zone_begins(s.model.actual["zones"])
    n1 = len(s.model.actual["zones"][1]["records"])
    rec = lambda k: dict(copy.deepcopy(pool[k % len(pool)]), name=f"edge{k}.{s.model.actual['zones'][0]['name']}")  # noqa: E731
    # zone 1's end and zone 3's (empty) front share nothing; zone 2's end and zone 3's front share rec_at == zb[3]: zone 2 first
    res, new_rows = s.records([(0, [(0, rec(0))]), (1, [(0, rec(1)), (n1, rec(2))]), (2, [(len(s.model.actual["zones"][2]["records"]), rec(3))]),
                               (3, [(0, rec(4)), (0, rec(5))]), (4, [(0, rec(6))])])
    at = [int(zb[0]), int(zb[1]), int(zb[2]), int(zb[3]), int(zb[3]), int(zb[3]), int(zb[4])]
    assert at[3] == at[4]  # the boundary case: the end of zone 2 is the front of zone 3
    assert new_rows == [a + k for k, a in enumerate(at)]
    names = [r["name"] for z in s.model.actual["zones"] for r in z["records"]]
    assert [names[r] for r in new_rows] == [rec(k)["name"] for k in range(7)]
    s.check()
    s.check_export()
    # delete plus insert at the same row (a replacement), deletes around it, and the resident row formula
    zb = zone_begins(s.model.actual["zones"])
    z = int(np.argmax(np.diff(zb)))
    r0 = int(zb[z]) + 1
    before = [r["name"] for zz in s.model.actual["zones"] for r in zz["records"]]
    res, new_rows = s.records([(z, [(1, rec(7))])], [r0, r0 + 1])
    after = [r["name"] for zz in s.model.actual["zones"] for r in zz["records"]]
    assert new_rows == [r0] and after[r0] == rec(7)["name"]
    for r in range(len(before)):
        if r not in (r0, r0 + 1):
            assert after[r - sum(1 for d in (r0, r0 + 1) if d < r) + (1 if r0 <= r else 0)] == before[r]
    s.check()
    # every record of a zone deleted; then an empty delta, which changes nothing
    zb = zone_begins(s.model.actual["zones"])
    s.records([], list(range(int(zb[z]), int(zb[z + 1]))))
    assert s.model.actual["zones"][z]["records"] == []
    s.check()
    s.check_export()
    n_rec, n_val = s.am.sizes()["n_records"], s.am.sizes()["n_values"]
    assert tuple(s.e.apply_records()) == (n_rec, n_val, 0, s.model.slab_len)
    s.check(rows=list(range(0, len(objects), 3)))


def test_hostsim_row_formulas_at_zone_ends(garecon, oracle, hostsim):
    edge_cases(garecon, oracle, hostsim)


# ------------------------------------------------------------------ refusals and state errors

BREAKAGES = ["at_next_zone", "at_range", "at_decreasing", "target_unsorted", "target_repeated", "target_range", "zone_name",
             "deleted_twice", "deleted_range", "csr", "lb_rows", "null_target", "null_at", "null_deleted"]


def refused_cases(garecon, engine, breakage):
    abi = garecon.abi
    objects, actual = randmodel.make(5, n_objects=20)
    zones = [z for z in actual["zones"]]
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    before = engine.diff()
    zb = zone_begins(zones)
    nz = len(zones)
    z0, z1 = [z for z in range(nz) if zb[z + 1] - zb[z] >= 2][:2]
    r = copy.deepcopy(zones[z0]["records"][0])
    packed = garecon.pack([], {"zones": [dict(zones[z0], records=[r, r]), dict(zones[z1], records=[r])]})
    args = dict(zone_target=[z0, z1], rec_at=[int(zb[z0]), int(zb[z0 + 1]), int(zb[z1]) + 1], deleted=[int(zb[z0])])
    if breakage == "at_next_zone":
        args["rec_at"] = [int(zb[z0]), int(zb[z0 + 1]) + 1, int(zb[z1]) + 1] if z1 == z0 + 1 else [int(zb[z0]), int(zb[z0 + 1]) + 1, int(zb[z1]) + 1]
    elif breakage == "at_range":
        args["rec_at"] = [int(zb[z0]), int(zb[z0]), int(zb[-1]) + 1]
    elif breakage == "at_decreasing":
        args["rec_at"] = [int(zb[z0]) + 1, int(zb[z0]), int(zb[z1])]
    elif breakage == "target_unsorted":
        packed = garecon.pack([], {"zones": [dict(zones[z1], records=[r, r]), dict(zones[z0], records=[r])]})
        args.update(zone_target=[z1, z0], rec_at=[int(zb[z1]), int(zb[z1]), int(zb[z0])])
    elif breakage == "target_repeated":
        packed = garecon.pack([], {"zones": [dict(zones[z0], records=[r, r]), dict(zones[z0], records=[r])]})
        args.update(zone_target=[z0, z0], rec_at=[int(zb[z0])] * 3)
    elif breakage == "target_range":
        args["zone_target"] = [z0, nz]
    elif breakage == "zone_name":
        packed = garecon.pack([], {"zones": [dict(zones[z0], records=[r, r]), dict(zones[z1], name="other.example.", records=[r])]})
    elif breakage == "deleted_twice":
        args["deleted"] = [1, 1]
    elif breakage == "deleted_range":
        args["deleted"] = [int(zb[-1])]
    elif breakage == "csr":
        packed.arrays["rec_val_begin"][1] = packed.arrays["rec_val_begin"][2] + 1
    elif breakage == "lb_rows":
        packed = garecon.pack([], {"zones": [dict(zones[z0], records=[r, r]), dict(zones[z1], records=[r])], "lbs": actual["lbs"][:1]})
    if breakage.startswith("null"):
        ok = np.asarray([z0, z1, 0], dtype=np.uint32)
        p = lambda a: a.ctypes.data_as(abi._u32p)  # noqa: E731
        d = abi.GarRecordDelta(ctypes.pointer(packed.actual), None if breakage == "null_target" else p(ok), None if breakage == "null_at" else p(ok), 1,
                               None if breakage == "null_deleted" else p(ok))
        assert engine.lib.gar_snapshot_apply_records(engine._h, ctypes.byref(d), ctypes.byref(abi.GarRecordDeltaResult())) == abi.GAR_E_INVALID
    else:
        with pytest.raises(garecon.GarError) as ei:
            engine.apply_records(packed.actual, **args)
        assert ei.value.rc == abi.GAR_E_INVALID, breakage
    assert engine.diff().diff(before) == []
    assert tuple(engine.apply_records()) == (int(snap.actual.n_records), int(snap.actual.n_values), 0, int(snap.actual.slab_len))
    assert engine.diff().diff(before) == []
    # the unbroken delta is accepted
    if breakage == "at_decreasing":
        packed = garecon.pack([], {"zones": [dict(zones[z0], records=[r, r]), dict(zones[z1], records=[r])]})
        engine.apply_records(packed.actual, [z0, z1], [int(zb[z0]), int(zb[z0 + 1]), int(zb[z1]) + 1], [int(zb[z0])])


@pytest.mark.parametrize("breakage", BREAKAGES)
def test_hostsim_invalid_record_delta_changes_nothing(garecon, hostsim, breakage):
    refused_cases(garecon, hostsim, breakage)


def test_hostsim_before_load_is_a_state_error(garecon):
    import __graft_entry__ as ge
    with garecon.Engine(cluster_name="default", lib=garecon.abi.load_library(ge.build_hostsim())) as e:
        for call in (lambda: e.apply_records(deleted=[0]), lambda: e.read_records([0])):
            with pytest.raises(garecon.GarError) as ei:
                call()
            assert ei.value.rc == garecon.abi.GAR_E_STATE


def test_ctypes_record_struct_sizes_match_header(garecon):
    src = textwrap.dedent('''
        #include <stdio.h>
        #include "garecon.h"
        int main(void) { printf("%zu %zu %zu\\n", sizeof(gar_record_delta), sizeof(gar_record_delta_result), sizeof(gar_record_readset)); return 0; }
    ''')
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(REPO / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout.split()
    abi = garecon.abi
    assert [int(x) for x in out] == [ctypes.sizeof(abi.GarRecordDelta), ctypes.sizeof(abi.GarRecordDeltaResult), ctypes.sizeof(abi.GarRecordReadSet)]


# ------------------------------------------------------------------ gar_read_records: the rule, restated

def owner_value(cluster, resource, key):
    return f'"heritage=aws-global-accelerator-controller,cluster={cluster},{resource}/{key}"'


def read_records_ref(objects, actual, cluster, rows, deleted=()):
    """The record rows gar_read_records reports (include/garecon.h), from the dict model: the records carrying an owner value of
    a key of the set, and the alias records of the same zone under their names."""
    vals = {owner_value(cluster, pyref._resource(objects[i]), f"{objects[i].get('ns', 'default')}/{objects[i]['name']}") for i in rows}
    vals |= {owner_value(cluster, "service" if kind == 0 else "ingress", key) for kind, key in deleted}
    out, g = [], 0
    for z in actual.get("zones", []):
        recs = z.get("records", [])
        owned = [any(v in vals for v in r.get("values", [])) for r in recs]
        names = {r["name"] for r, o in zip(recs, owned) if o}
        out += [g + k for k, r in enumerate(recs) if owned[k] or (r.get("alias") is not None and r["name"] in names)]
        g += len(recs)
    return out


def check_exact(garecon, e, objects, actual, seed, deleted=()):
    trs.load(garecon, e, objects, actual)
    zb = zone_begins(actual.get("zones", []))
    rng = random.Random(seed)
    for rows, dk in trs.keysets(objects, actual, rng, trs.deleted_keys(objects, actual, deleted)):
        got = e.read_records(rows, dk)
        assert np.all(got[1:] > got[:-1])
        assert got.tolist() == read_records_ref(objects, actual, "default", rows, dk), (len(rows), len(dk))
        zones = set(trs.got(e, rows, dk)["zones"])
        assert set((np.searchsorted(zb, got, side="right") - 1).tolist()) <= zones  # inside the zones gar_read_set reports


@pytest.mark.parametrize("seed", range(6))
def test_exact_randmodel(garecon, eng, seed):
    objects, actual, dropped = scalemodels.randmodel_dropped(seed, 300)
    check_exact(garecon, eng, objects, actual, seed, dropped)


@pytest.mark.parametrize("seed", range(3))
def test_exact_multilbi_and_hot(garecon, eng, seed):
    check_exact(garecon, eng, *multilbi.make(seed, n_objects=50), seed)
    objects, actual = scalemodels.hot_cluster(seed, 300)
    check_exact(garecon, eng, objects, actual, seed, [scalemodels.key_of(ob) for ob in objects[:3]])
    objects, actual = hotkeys.make()
    check_exact(garecon, eng, objects, actual, seed, [scalemodels.key_of(ob) for ob in objects[:2]])


def test_read_records_leaves_state_and_replay(garecon, eng):
    objects, actual, dropped = scalemodels.randmodel_dropped(7, 300)
    trs.load(garecon, eng, objects, actual)
    for _ in range(4):
        eng.diff()
    mode = eng.counters()["launch_mode"]
    before = trs.export_bytes(eng)
    rows = list(range(0, len(objects), 7))
    first = eng.read_records(rows, dropped[:5])
    assert np.array_equal(eng.read_records(rows, dropped[:5]), first)
    assert trs.export_bytes(eng) == before
    eng.diff()
    assert eng.counters()["launch_mode"] == mode
    assert eng.read_set(rows, dropped[:5]).zone_rows.tolist() == trs.want(objects, actual, rows, dropped[:5])["zones"]  # unchanged
    for bad in ([len(objects)], [0, 1 << 31]):
        with pytest.raises(garecon.abi.GarError) as ei:
            eng.read_records(bad)
        assert ei.value.rc == -1
    assert eng.read_records([]).size == 0


# ------------------------------------------------------------------ sufficiency

def renumber(cs, rec_map, val_map):
    """The ops of a change set with record and value rows mapped to their rows after a record delta."""
    out = []
    for op in cs.ops.tolist():
        op = list(op)
        code = op[0] & 0xFF
        if code == R53_UPSERT_A and op[5] < 0xFFFFFFFE:
            op[5] = rec_map[op[5]]
        elif code == R53_DELETE_RECORD:
            op[4], op[5] = rec_map[op[4]], val_map[op[5]]
        out.append(op)
    return out


def check_sufficiency(garecon, e, objects, actual, seed, deleted):
    rng = random.Random(seed)
    n = len(objects)
    rows = rng.sample(range(n), max(1, n // rng.choice([2, 10, 50])))
    dk = rng.sample(deleted, min(len(deleted), 5)) + [(0, "default/absent")]
    snap = trs.load(garecon, e, objects, actual)
    before = e.diff_keys(rows, dk)
    keep = set(e.read_records(rows, dk).tolist())
    zones = actual["zones"]
    zb = zone_begins(zones)
    # every record outside the set: rewritten (fresh name, values that are no owner value, maybe an alias), deleted or kept; fresh
    # records inserted in front of every kind of row and at zone ends
    inserts, deleted_rows, serial = [], [], 0
    for z, zone in enumerate(zones):
        ins = []
        for p, rec in enumerate(zone.get("records", [])):
            if rng.random() < 0.3:
                serial += 1
                ins.append((p, {"name": f"q{serial}.{zone['name']}", "type": rng.choice(["A", "TXT"]), "values": [f'"w{serial}"']}))
            if zb[z] + p in keep:
                continue
            c = rng.random()
            if c < 0.4:
                deleted_rows.append(int(zb[z]) + p)
                serial += 1
                nr = {"name": f"q{serial}.{zone['name']}", "type": rng.choice(["A", "TXT"]), "values": [f'"w{serial}.{x}"' for x in range(rng.randrange(0, 3))]}
                if rng.random() < 0.3:
                    nr["alias"] = f"z{serial}.awsglobalaccelerator.com."
                ins.append((p, nr))
            elif c < 0.7:
                deleted_rows.append(int(zb[z]) + p)
        if rng.random() < 0.5:
            serial += 1
            ins.append((len(zone.get("records", [])), {"name": f"q{serial}.{zone['name']}", "type": "TXT", "values": [f'"w{serial}"']}))
        inserts.append((z, ins))
    inserts = [(z, ins) for z, ins in inserts if ins]
    packed = garecon.pack([], {"zones": [dict(zones[z], records=[r for _, r in ins]) for z, ins in inserts]}) if inserts else None
    trs._alive[id(e)].append(packed)
    at = [int(zb[z]) + p for z, ins in inserts for p, _ in ins]
    e.apply_records(packed.actual if packed else None, [z for z, _ in inserts], at, deleted_rows)
    after = e.diff_keys(rows, dk)
    # the row formulas give the new record rows; values follow their records
    dl, at_a = np.sort(np.asarray(deleted_rows, dtype=np.int64)), np.asarray(at, dtype=np.int64)
    old = np.arange(int(zb[-1]))
    new = old - np.searchsorted(dl, old) + np.searchsorted(at_a, old, side="right")
    x = e.export(ACT)
    nb = garecon.tables.columns(x.actual, garecon.tables.ACT_TABLES)["rec_val_begin"].astype(np.int64)
    ob = np.asarray(snap.arrays["rec_val_begin"]).astype(np.int64)
    val_map = {}
    for r in keep:
        for v in range(ob[r], ob[r + 1]):
            val_map[v] = int(nb[new[r]] + v - ob[r])
    assert after.ops.shape == before.ops.shape
    assert renumber(before, {r: int(new[r]) for r in keep}, val_map) == [list(op) for op in after.ops.tolist()]
    for k in ("status_ga", "status_r53", "derived"):
        assert np.array_equal(getattr(after, k), getattr(before, k)), k


@pytest.mark.parametrize("seed", range(10))
def test_sufficiency(garecon, hostsim, seed):
    objects, actual, dropped = scalemodels.randmodel_dropped(seed, 120)
    check_sufficiency(garecon, hostsim, objects, actual, seed, dropped)


@pytest.mark.parametrize("seed", range(2))
def test_sufficiency_multilbi_hot(garecon, hostsim, seed):
    check_sufficiency(garecon, hostsim, *multilbi.make(seed, n_objects=60), seed, [])
    objects, actual = scalemodels.hot_cluster(seed, 200)
    check_sufficiency(garecon, hostsim, objects, actual, seed, [scalemodels.key_of(ob) for ob in objects[:4]])


# ------------------------------------------------------------------ the refresh loop at record granularity

def record_ids(garecon, e):
    """(zone, name, type, ordinal) of every resident record row and (record id, index) of every value row, from an export."""
    x = e.export(ACT)
    c = garecon.tables.columns(x.actual, garecon.tables.ACT_TABLES)
    slab = np.asarray(c["slab"]).tobytes()
    zb, vb = c["zone_rec_begin"].astype(np.int64), c["rec_val_begin"].astype(np.int64)
    rec, val, seen = [], [], {}
    for z in range(len(zb) - 1):
        for r in range(zb[z], zb[z + 1]):
            ref = int(c["rec_name"][r])
            k = (z, slab[ref & ((1 << 40) - 1):][:ref >> 40], int(c["rec_type"][r]))
            seen[k] = seen.get(k, -1) + 1
            rec.append(k + (seen[k],))
            val += [(rec[-1], v - vb[r]) for v in range(vb[r], vb[r + 1])]
    return rec, val


def by_identity(garecon, e, cs):
    rec, val = record_ids(garecon, e)
    return renumber(cs, rec, val), cs.status_ga.tolist(), cs.status_r53.tolist()


def record_refresh(garecon, e, cloud_cols, rows, deleted=()):
    """The worker loop at record granularity: read set (LBs, accelerators) + record read set -> re-describe -> two deltas."""
    rs = trs.got(e, rows, deleted)
    d = {"lbs": [(r, cloud_cols["dict"]["lbs"][r]) for r in rs["lbs"]], "accs": [(r, cloud_cols["dict"]["accelerators"][r]) for r in rs["accs"]], "zones": []}
    trs.apply_rows(garecon, e, cloud_cols["dict"], d)
    rr = e.read_records(rows, deleted)
    x = e.export(ACT)
    resident = garecon.tables.columns(x.actual, garecon.tables.ACT_TABLES)
    delta = deltas_mod().record_refresh(resident, cloud_cols["cols"], rr)
    keep = deltas_mod().actual_struct(delta["rows"]) if delta["rows"] is not None else (None, None)
    trs._alive[id(e)] += [x, keep]
    e.apply_records(keep[1], delta["zone_target"], delta["rec_at"], delta["deleted"])


def refresh_case(garecon, oracle, eng, seed):
    """Owned alias targets changed, some alias records and owned metadata sets deleted in the cloud: the zone-granular and the
    record-granular refresh loops reach the same change sets, record for record."""
    objects, stale, dropped = scalemodels.randmodel_dropped(seed, 200)
    cloud = copy.deepcopy(stale)
    rng = random.Random(seed)
    for z in cloud["zones"]:
        recs = []
        for r in z.get("records", []):
            if r.get("alias") is not None:
                c = rng.random()
                if c < 0.3:
                    continue
                if c < 0.6:
                    r["alias"] = "moved.awsglobalaccelerator.com."
            elif rng.random() < 0.1:
                continue
            recs.append(r)
        z["records"] = recs
    csnap = garecon.pack([], cloud)
    cloud_cols = {"dict": cloud, "cols": garecon.tables.columns(csnap.actual, garecon.tables.ACT_TABLES)}
    rows = rng.sample(range(len(objects)), len(objects) // 3)
    dk = dropped[:5]
    trs.load(garecon, eng, objects, stale)
    trs.refresh(garecon, eng, cloud, rows, dk)
    zone_loop = by_identity(garecon, eng, eng.diff_keys(rows, dk))
    assert eng.diff_keys(rows, dk).diff(oracle.diff_keys(garecon.pack(objects, cloud), rows, dk, mode=0)) == []
    trs.load(garecon, eng, objects, stale)
    trs._alive[id(eng)].append(csnap)
    record_refresh(garecon, eng, cloud_cols, rows, dk)
    rec_loop = by_identity(garecon, eng, eng.diff_keys(rows, dk))
    assert rec_loop == zone_loop


@pytest.mark.parametrize("seed", range(4))
def test_refresh_loop_at_record_granularity(garecon, oracle, eng, seed):
    refresh_case(garecon, oracle, eng, seed)


# ------------------------------------------------------------------ GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(700, 708))
def test_gpu_random_sequences(garecon, oracle, engine, seed):
    run_sequence(garecon, oracle, engine, seed, n_objects=80, n_batches=random.Random(seed).randrange(4, 9), oracle_mode=1)


@pytest.mark.gpu
def test_gpu_edges_refusals_and_state_errors(garecon, oracle, engine):
    edge_cases(garecon, oracle, engine)
    for breakage in BREAKAGES:
        refused_cases(garecon, engine, breakage)
    with garecon.Engine(cluster_name="default") as e:
        for call in (lambda: e.apply_records(deleted=[0]), lambda: e.read_records([0])):
            with pytest.raises(garecon.GarError) as ei:
                call()
            assert ei.value.rc == garecon.abi.GAR_E_STATE
        objects, actual = randmodel.make(5, n_objects=20)
        e.load(garecon.pack(objects, actual))
        e.shard_route(garecon.abi.GarShard(0, 1, 0, 0, 0, 0, 0, 0, 0), 1)
        for call in (lambda: e.apply_records(deleted=[0]), lambda: e.read_records([0])):
            with pytest.raises(garecon.GarError) as ei:
                call()
            assert ei.value.rc == garecon.abi.GAR_E_STATE


@pytest.mark.gpu
def test_gpu_attached_is_a_state_error(garecon):
    import torch
    tables = garecon.tables
    objects, actual = randmodel.make(5, n_objects=20)
    snap = garecon.pack(objects, actual)
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
            e.apply_records(deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE
        assert e.diff().diff(before) == []
        assert e.read_records([0, 1]).tolist() == read_records_ref(objects, actual, "default", [0, 1])  # reading an attached snapshot is allowed


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(2))
def test_gpu_read_records_scale(garecon, engine, seed):
    objects, actual, dropped = scalemodels.randmodel_dropped(seed, 20000)
    check_exact(garecon, engine, objects, actual, seed, dropped[:100])
    objects, actual = scalemodels.hot_cluster(seed, 20000)
    check_exact(garecon, engine, objects, actual, seed)


@pytest.mark.gpu
def test_gpu_sufficiency(garecon, engine):
    objects, actual, dropped = scalemodels.randmodel_dropped(3, 5000)
    check_sufficiency(garecon, engine, objects, actual, 3, dropped)


@pytest.mark.gpu
def test_gpu_hot_owner(garecon, engine):
    """One key owning 10^5 owner values in 10^5 TXT sets, each with an alias record under its name: 2 * 10^5 + 1 rows."""
    n = 100_000
    hot = {"kind": "service", "ns": "default", "name": "hot", "lb_ingress": [], "annotations": {}}
    cold = {"kind": "service", "ns": "default", "name": "cold", "lb_ingress": [], "annotations": {}}
    recs = []
    for k in range(n):
        recs.append({"name": f"r{k}.example.com.", "type": "TXT", "values": [owner_value("default", "service", "default/hot")]})
        recs.append({"name": f"r{k}.example.com.", "type": "A", "alias": f"a{k}.awsglobalaccelerator.com.", "values": []})
    recs.append({"name": "c.example.com.", "type": "TXT", "values": [owner_value("default", "service", "default/cold")]})
    actual = {"lbs": [], "accelerators": [], "zones": [{"name": "example.com.", "records": recs}]}
    trs.load(garecon, engine, [hot, cold], actual)
    assert engine.read_records([0]).tolist() == list(range(2 * n))
    assert engine.read_records([1]).tolist() == [2 * n]
    assert engine.read_records([], [(0, "default/hot")]).tolist() == list(range(2 * n))


def splice_at(m, rows_at, rng):
    """A record delta over a column mirror: the resident rows `rows_at` deleted and each replaced by a copy of a random record,
    plus one copy inserted in front of each."""
    cur = m.cur
    zb = np.asarray(cur["zone_rec_begin"]).astype(np.int64)
    n_rec = int(zb[-1])
    rows_at = sorted(rows_at)
    zones = np.searchsorted(zb, rows_at, side="right") - 1
    by_zone = {}
    for r, z in zip(rows_at, zones.tolist()):
        by_zone.setdefault(z, []).extend([(r, int(rng.integers(0, n_rec))), (r, int(rng.integers(0, n_rec)))])
    zs = sorted(by_zone)
    return dict(rows=deltas_mod().record_rows(cur, zs, [[s for _, s in by_zone[z]] for z in zs]), zone_target=np.asarray(zs, dtype=np.uint32),
                rec_at=np.asarray([r for z in zs for r, _ in by_zone[z]], dtype=np.uint32), deleted=np.asarray(rows_at, dtype=np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("n_objects", [20000, 60000])
def test_gpu_scale_tile_boundaries(garecon, oracle, engine, n_objects):
    """Splices across scan-tile boundaries (rows 2047 / 2048 / 4095 / 4096 deleted and inserted) and record_churn batches on the
    scale models: after each, the full diff equals a fresh load of the mirrored tables, and keyed diffs the oracle."""
    deltas, tables = deltas_mod(), garecon.tables
    objects, actual, dropped = scalemodels.randmodel_dropped(n_objects % 7, n_objects)
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    engine.diff()
    m = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    o_cols = tables.columns(snap.objects, tables.OBJ_TABLES)
    rng = np.random.default_rng(n_objects)
    assert m.sizes()["n_records"] > 4097
    arms = [lambda: splice_at(m, [2047, 2048, 4095, 4096], rng), lambda: deltas.record_churn(m, rng, n_zones=50, per_zone=20),
            lambda: deltas.record_redescribe(m.cur, engine.read_records(list(range(0, len(objects), 5)), dropped[:50]))]
    with garecon.Engine(cluster_name="default") as fresh:
        for arm in arms:
            d = arm()
            keep, rows = deltas.actual_struct(d["rows"]) if d["rows"] is not None else (None, None)
            res = engine.apply_records(rows, d["zone_target"], d["rec_at"], d["deleted"])
            want = m.apply_records(**d)
            assert tuple(res) == tuple(want[k] for k in garecon.abi.RecordDeltaResult.FIELDS)
            msnap = m.snapshot(o_cols)
            fresh.load(msnap)
            got, ref = engine.diff(), fresh.diff()
            assert got.diff(ref) == [], got.describe_first_mismatch(ref)
            ks = list(range(0, len(objects), 11))
            assert engine.diff_keys(ks, dropped[:20]).diff(fresh.diff_keys(ks, dropped[:20])) == []
            assert np.array_equal(engine.read_records(ks, dropped[:20]), fresh.read_records(ks, dropped[:20]))
    want = oracle.diff_keys(msnap, ks, dropped[:20], mode=1)
    got = engine.diff_keys(ks, dropped[:20])
    assert got.diff(want) == [], got.describe_first_mismatch(want)


@pytest.mark.gpu
@pytest.mark.parametrize("no_graph", [False, True])
def test_gpu_replay_after_record_delta(garecon, monkeypatch, no_graph):
    """After a record delta the recording of the old tables is never replayed: full diffs go eager, record (1), replay (2), equal
    to a fresh load throughout; with GAR_NO_GRAPH=1 the same answers, never recorded."""
    from test_launch_replay import _engine
    deltas, tables = deltas_mod(), garecon.tables
    objects, actual = randmodel.make(4, n_objects=80)
    snap = garecon.pack(objects, actual)
    results = []
    with _engine(garecon, monkeypatch, no_graph) as e, garecon.Engine(cluster_name="default") as fresh:
        e.load(snap)
        for _ in range(4):
            e.diff()
        m = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
        rng = np.random.default_rng(4)
        for _ in range(2):
            d = deltas.record_churn(m, rng)
            keep, rows = deltas.actual_struct(d["rows"]) if d["rows"] is not None else (None, None)
            e.apply_records(rows, d["zone_target"], d["rec_at"], d["deleted"])
            m.apply_records(**d)
            fresh.load(m.snapshot(tables.columns(snap.objects, tables.OBJ_TABLES)))
            ref = fresh.diff()
            modes = []
            for _ in range(4):
                cs = e.diff()
                assert cs.diff(ref) == [], cs.describe_first_mismatch(ref)
                modes.append(e.counters()["launch_mode"])
            results.append(modes)
    for modes in results:
        if no_graph:
            assert modes == [0, 0, 0, 0]
        else:
            assert modes[0] == 0 and modes[-2:] == [1, 2], modes


@pytest.mark.gpu
def test_gpu_record_loop_at_scale(garecon, oracle, engine):
    """configs[2] at 10^6 objects, the worker's loop at record granularity with a churned cloud: read set + record read set ->
    re-described rows (LBs, accelerators, record sets) -> apply_actual + apply_records; the keyed change set equals a fresh load's
    of the resulting tables, and the full diff too."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    deltas, tables = deltas_mod(), garecon.tables
    snap = synth.generate(3, 1_000_000)
    engine.load(snap)
    m = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    o_cols = tables.columns(snap.objects, tables.OBJ_TABLES)
    rng = np.random.default_rng(9)
    d = deltas.record_churn(m, rng, n_zones=40, per_zone=50)  # the cloud moved on: record sets replaced, inserted, deleted
    keep, rows = deltas.actual_struct(d["rows"]) if d["rows"] is not None else (None, None)
    engine.apply_records(rows, d["zone_target"], d["rec_at"], d["deleted"])
    m.apply_records(**d)
    n = int(snap.objects.n_objects)
    ks = random.Random(9).sample(range(n), 10_000)
    rs = engine.read_set(ks)
    a = deltas.compact_actual(deltas.actual_rows(m.cur, rs.lb_rows, rs.acc_rows))
    keep_a, arows = deltas.actual_struct(a)
    engine.apply_actual(arows, rs.lb_rows, rs.acc_rows)
    m.apply(a, rs.lb_rows, rs.acc_rows)
    rr = engine.read_records(ks)
    r = deltas.record_redescribe(m.cur, rr)
    keep_r, rrows = deltas.actual_struct(r["rows"])
    engine.apply_records(rrows, r["zone_target"], r["rec_at"], r["deleted"])
    m.apply_records(**r)
    got = engine.diff_keys(ks)
    with garecon.Engine(cluster_name=snap.cluster) as fresh:
        fresh.load(m.snapshot(o_cols))
        ref = fresh.diff_keys(ks)
        assert got.diff(ref) == [], got.describe_first_mismatch(ref)
        full, ref_full = engine.diff(), fresh.diff()
        assert full.diff(ref_full) == [], full.describe_first_mismatch(ref_full)
