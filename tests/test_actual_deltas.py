"""AWS deltas (gar_snapshot_apply_actual): re-listed load balancers, accelerator subtrees and zone record lists applied to the
resident AWS tables.  After every delta the engine must answer exactly as a fresh gar_snapshot_load of the AWS model a small
Python model of the rules holds (include/garecon.h "AWS deltas"), against the oracle: full diff, incremental diff and the
EndpointGroupBinding set-diff.  AWS and object deltas interleave.  The change set holds no AWS-slab references, so every array
but tok_name / tok_region (object-slab references, compared as the strings they name) is compared bit for bit."""
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
from test_convergence import _rounds
from test_object_deltas import Events, Mirror, assert_same_full, key_of

REPO = Path(__file__).resolve().parent.parent
NONE = 0xFFFFFFFF


def deltas_mod():
    return importlib.import_module("aws-global-accelerator-controller_b200.deltas")


class AwsModel:
    """The rules of include/garecon.h "AWS deltas" on the dict model of tables.pack, plus the resident AWS slab length."""

    def __init__(self, actual, snap):
        self.actual = copy.deepcopy(actual)
        self.actual.setdefault("lbs", [])
        self.actual.setdefault("accelerators", [])
        self.actual.setdefault("zones", [])
        self.slab_len = int(snap.actual.slab_len)

    def apply(self, d):
        """d: {"lbs": [(target, lb)], "accs": [(target, acc)], "zones": [(zone row, records)], "lb_deleted": [...],
        "acc_deleted": [...]}.  -> the expected result tuple of Engine.apply_actual."""
        a = self.actual
        for key, tkey, dkey in (("lbs", "lbs", "lb_deleted"), ("accelerators", "accs", "acc_deleted")):
            old = a[key]
            repl = {t: x for t, x in d.get(tkey, []) if t != NONE}
            gone = set(d.get(dkey, []))
            a[key] = [repl.get(r, x) for r, x in enumerate(old) if r not in gone] + [x for t, x in d.get(tkey, []) if t == NONE]
        for z, recs in d.get("zones", []):
            a["zones"][z] = dict(a["zones"][z], records=recs)
        base = 0
        if d.get("lbs") or d.get("accs") or d.get("zones"):
            base = (self.slab_len + 15) & ~15
            self.slab_len = base + int(d["_rows"].actual.slab_len)
        return self.expected(base)

    def expected(self, base):
        a = self.actual
        lis = [li for x in a["accelerators"] for li in x.get("listeners", [])]
        egs = [eg for li in lis for eg in li.get("egs", [])]
        recs = [r for z in a["zones"] for r in z.get("records", [])]
        return (len(a["lbs"]), len(a["accelerators"]), sum(len(x.get("tags", [])) for x in a["accelerators"]), len(lis),
                sum(len(li.get("ports", [])) for li in lis), len(egs), sum(len(eg.get("endpoints", [])) for eg in egs), len(recs),
                sum(len(r.get("values", [])) for r in recs), base, self.slab_len)


def apply_delta(garecon, engine, model, d):
    """Pack delta d (AwsModel.apply's form), apply it to the engine and the model; check the result."""
    rows = {"lbs": [x for _, x in d.get("lbs", [])], "accelerators": [x for _, x in d.get("accs", [])],
            "zones": [dict(model.actual["zones"][z], records=r) for z, r in d.get("zones", [])]}
    has_rows = any(rows.values())
    d["_rows"] = garecon.pack([], rows) if has_rows else None
    res = engine.apply_actual(d["_rows"].actual if has_rows else None, [t for t, _ in d.get("lbs", [])], [t for t, _ in d.get("accs", [])],
                              [z for z, _ in d.get("zones", [])], d.get("lb_deleted", []), d.get("acc_deleted", []))
    want = model.apply(d)
    assert tuple(res) == want, (tuple(res), want)
    return res


class AwsEvents:
    """Random re-list results over a randmodel AWS model: LB replace (state, DNS) / append (duplicate (region, name)) / delete,
    accelerator replace (another subtree: 0, 1 or many listeners, EGs, endpoints, tags) / append / delete, and zone record
    lists replaced (empty, reordered, a record dropped, a multi-value TXT set)."""

    def __init__(self, seed):
        self.rng = random.Random(seed * 131 + 7)
        pool_actual = randmodel.make(seed + 7000, n_objects=30)[1]
        self.acc_pool = pool_actual.get("accelerators", []) + [
            {"name": "bare", "dns": "bare.awsglobalaccelerator.com", "enabled": False, "tags": [], "listeners": []},
            {"name": "wide", "dns": "wide.awsglobalaccelerator.com", "tags": [("k", "v")] * 3,
             "listeners": [{"proto": "UDP", "ports": [53, 54], "egs": [{"endpoints": ["e1", "e2", "e3"]}, {"endpoints": []}]},
                           {"proto": "TCP", "ports": [], "egs": []}]}]

    def batch(self, actual):
        rng = self.rng
        d = {"lbs": [], "accs": [], "zones": [], "lb_deleted": [], "acc_deleted": []}
        lbs, accs, zones = actual["lbs"], actual["accelerators"], actual["zones"]
        rows = list(range(len(lbs)))
        rng.shuffle(rows)
        for r in rows[:rng.randrange(0, 4)]:
            if rng.random() < 0.35:
                d["lb_deleted"].append(r)  # often a row ahead of a duplicate (region, name): the later row must win next
            else:
                lb = dict(lbs[r], state=rng.choice(["active", "provisioning", "failed", "active_impaired"]))
                if rng.random() < 0.3:
                    lb["dns"] = rng.choice(lbs)["dns"]
                d["lbs"].append((r, lb))
        for _ in range(rng.randrange(0, 3)):
            if lbs:
                d["lbs"].append((NONE, dict(rng.choice(lbs), dns="dup-" + rng.choice(lbs)["dns"], state=rng.choice(["active", "provisioning"]))))
        rows = list(range(len(accs)))
        rng.shuffle(rows)
        for r in rows[:rng.randrange(0, 5)]:
            if rng.random() < 0.3:
                d["acc_deleted"].append(r)
            else:
                new = copy.deepcopy(rng.choice(accs + self.acc_pool))
                if rng.random() < 0.5:  # the same accelerator, re-described after the worker changed it
                    new = copy.deepcopy(accs[r])
                    for li in new.get("listeners", []):
                        li["ports"] = [rng.choice([80, 443, 8080])] + li.get("ports", [])[1:]
                        for eg in li.get("egs", []):
                            eg["endpoints"] = rng.sample([x["arn"] for x in lbs], min(len(lbs), rng.randrange(0, 3)))
                d["accs"].append((r, new))
        for _ in range(rng.randrange(0, 3)):
            d["accs"].append((NONE, copy.deepcopy(rng.choice(accs + self.acc_pool))))
        for z in rng.sample(range(len(zones)), min(len(zones), rng.randrange(0, 3))):
            recs = copy.deepcopy(zones[z].get("records", []))
            c = rng.randrange(4)
            if c == 0:
                recs = []
            elif c == 1:
                rng.shuffle(recs)
            elif c == 2 and recs:
                recs.pop(rng.randrange(len(recs)))
            else:
                recs.append({"name": f"txt{rng.randrange(99)}.{zones[z]['name']}", "type": "TXT",
                             "values": [f'"v{i}"' for i in range(rng.randrange(2, 40))]})
            d["zones"].append((z, recs))
        return d


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


def check_all(garecon, oracle, engine, omirror, model, bindings, rows, deleted, oracle_mode):
    msnap = garecon.pack(omirror.objects, model.actual)
    got = engine.diff_keys(rows, deleted)
    want = oracle.diff_keys(msnap, rows, deleted, mode=oracle_mode)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert_same_full(engine.diff(), oracle.diff(msnap, "default", mode=1), omirror.slab, msnap.arrays["o.slab"])
    assert engine.bindings_diff(bindings).ops.tolist() == oracle.bindings_diff(msnap, bindings).ops.tolist()


def run_sequence(garecon, oracle, engine, seed, n_objects, n_batches, oracle_mode):
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=n_objects, n_bindings=3 * n_objects)
    snap = garecon.pack(objects, actual)
    b = garecon.pack_bindings(bindings, known)
    engine.load(snap)
    omirror, model = Mirror(objects, snap), AwsModel(actual, snap)
    oevents, aevents = Events(seed, actual), AwsEvents(seed)
    rng = random.Random(seed)
    if seed % 3 == 0:
        engine.diff()
    for _ in range(n_batches):
        if rng.random() < 0.4:  # an object delta between AWS deltas
            upserts, deleted = oevents.batch(omirror.objects)
            usnap = garecon.pack(upserts, None) if upserts else None
            engine.apply_objects(usnap.objects if usnap else None, deleted)
            omirror.apply(upserts, deleted, usnap)
        apply_delta(garecon, engine, model, aevents.batch(model.actual))
        rows = rng.sample(range(len(omirror.objects)), min(len(omirror.objects), 8))
        deleted = [key_of(o) for o in rng.sample(objects, 2)] if rng.random() < 0.5 else []
        deleted = [k for k in deleted if k not in {key_of(o) for o in omirror.objects}]
        check_all(garecon, oracle, engine, omirror, model, b, rows, deleted, oracle_mode)


@pytest.mark.parametrize("seed", range(20))
def test_hostsim_random_sequences(garecon, oracle, hostsim, seed):
    run_sequence(garecon, oracle, hostsim, seed, n_objects=30, n_batches=random.Random(seed).randrange(4, 9), oracle_mode=0)


def test_hostsim_sequence_with_tiny_capacities(garecon, oracle, hostsim, monkeypatch):
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    run_sequence(garecon, oracle, hostsim, 103, n_objects=30, n_batches=5, oracle_mode=0)


def test_hostsim_first_row_wins_after_deletes_ahead(garecon, oracle, hostsim):
    """Duplicate (region, name) LB rows: deleting the first makes the second one the answer; replacing it keeps its place."""
    objects, actual = randmodel.make(21, n_objects=20)
    lbs = actual["lbs"]
    actual["lbs"] = [dict(lb, dns="first-" + lb["dns"]) for lb in lbs] + lbs  # every (region, name) twice; the first row is wrong
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    model, om = AwsModel(actual, snap), Mirror(objects, snap)
    n = len(lbs)
    for d in ({"lb_deleted": list(range(0, n, 2))}, {"lbs": [(0, dict(lbs[0], state="provisioning"))]}, {"lb_deleted": [0]}):
        apply_delta(garecon, hostsim, model, d)
        msnap = garecon.pack(om.objects, model.actual)
        assert_same_full(hostsim.diff(), oracle.diff(msnap, "default", mode=1), om.slab, msnap.arrays["o.slab"])


def model_delta(old, new):
    """The AWS delta that turns model `old` into `new` after tests/executor.py ran: LBs by position, accelerators by arn
    (deletes keep order, creates are appended), zones by position (replaced when the record list differs)."""
    d = {"lbs": [], "accs": [], "zones": [], "lb_deleted": [], "acc_deleted": []}
    ol, nl = old.get("lbs", []), new.get("lbs", [])
    d["lbs"] = [(i, nl[i]) for i in range(min(len(ol), len(nl))) if ol[i] != nl[i]] + [(NONE, x) for x in nl[len(ol):]]
    d["lb_deleted"] = list(range(len(nl), len(ol)))
    oa, na = old.get("accelerators", []), new.get("accelerators", [])
    # the new list is the surviving old rows in order, then the created ones; the executor numbers created ARNs per round, so
    # align greedily (any alignment of that shape yields the same table)
    surv, o = [], 0
    for i, x in enumerate(na):
        r = next((r for r in range(o, len(oa)) if oa[r]["arn"] == x["arn"]), None)
        if r is None:
            break
        surv.append((r, i))
        o = r + 1
    kept = {r for r, _ in surv}
    d["acc_deleted"] = [r for r in range(len(oa)) if r not in kept]
    d["accs"] = [(r, na[i]) for r, i in surv if na[i] != oa[r]] + [(NONE, x) for x in na[len(surv):]]
    d["zones"] = [(z, new["zones"][z].get("records", [])) for z in range(len(old.get("zones", []))) if old["zones"][z].get("records", []) != new["zones"][z].get("records", [])]
    return d


def converge(garecon, oracle, engine, seed, oracle_mode):
    objects, actual = randmodel.make(seed, n_objects=40)
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    model, om = AwsModel(actual, snap), Mirror(objects, snap)
    state = {"actual": copy.deepcopy(actual), "first": True}

    def diff_fn(s):
        cur = s.model[1]
        if not state["first"]:
            apply_delta(garecon, engine, model, model_delta(state["actual"], cur))
        state["first"] = False
        state["actual"] = copy.deepcopy(cur)
        got = engine.diff()
        want = oracle.diff(garecon.pack(objects, cur), "default", mode=1)
        assert_same_full(got, want, om.slab, s.arrays["o.slab"])
        return got

    hist = _rounds(garecon, objects, actual, diff_fn)
    ref = _rounds(garecon, objects, actual, lambda s: oracle.diff(s, "default", mode=1))
    assert [h.ops.tolist() for h in hist] == [h.ops.tolist() for h in ref]


@pytest.mark.parametrize("seed", range(6))
def test_hostsim_converges_without_reload(garecon, oracle, hostsim, seed):
    converge(garecon, oracle, hostsim, seed, 0)


def _small(garecon, seed=5):
    objects, actual = randmodel.make(seed, n_objects=20)
    return objects, actual, garecon.pack(objects, actual)


@pytest.mark.parametrize("breakage", ["lb_range", "acc_range", "zone_range", "replace_and_delete", "twice", "zone_twice", "zone_name", "csr",
                                      "string", "enum", "null_target", "null_deleted"])
def test_hostsim_invalid_delta_changes_nothing(garecon, oracle, hostsim, breakage):
    objects, actual, snap = _small(garecon)
    hostsim.load(snap)
    before = hostsim.diff()
    abi = garecon.abi
    lb, acc, z = actual["lbs"][0], actual["accelerators"][0], actual["zones"][0]
    rows = garecon.pack([], {"lbs": [lb], "accelerators": [acc], "zones": [z]})
    args = dict(lb_target=[0], acc_target=[0], zone_target=[0], lb_deleted=[], acc_deleted=[])
    if breakage == "lb_range":
        args["lb_target"] = [len(actual["lbs"])]
    elif breakage == "acc_range":
        args["acc_deleted"] = [len(actual["accelerators"])]
    elif breakage == "zone_range":
        args["zone_target"] = [len(actual["zones"])]
    elif breakage == "replace_and_delete":
        args["acc_deleted"] = [0]
    elif breakage == "twice":
        args["lb_deleted"] = [1, 1]
    elif breakage == "zone_twice":
        rows = garecon.pack([], {"lbs": [lb], "accelerators": [acc], "zones": [z, z]})
        args["zone_target"] = [0, 0]
    elif breakage == "zone_name":
        args["zone_target"] = [next(i for i, x in enumerate(actual["zones"]) if x["name"] != z["name"])]
    elif breakage == "csr":
        rows.arrays["acc_lis_begin"][0] = 1
    elif breakage == "string":
        rows.arrays["lb_dns"][0] = (4 << 40) | int(rows.actual.slab_len)
    elif breakage == "enum":
        rows.arrays["lb_state"][0] = 4
    if breakage.startswith("null"):
        d = abi.GarActualDelta(ctypes.pointer(rows.actual), None if breakage == "null_target" else rows.arrays["acc_lis_begin"].ctypes.data_as(abi._u32p),
                               rows.arrays["acc_lis_begin"].ctypes.data_as(abi._u32p), rows.arrays["acc_lis_begin"].ctypes.data_as(abi._u32p), 1, None, 0, None)
        res = abi.GarActualDeltaResult()
        rc = hostsim.lib.gar_snapshot_apply_actual(hostsim._h, ctypes.byref(d), ctypes.byref(res))
        assert rc == abi.GAR_E_INVALID
    else:
        with pytest.raises(garecon.GarError) as ei:
            hostsim.apply_actual(rows.actual, **args)
        assert ei.value.rc == abi.GAR_E_INVALID
    assert hostsim.diff().diff(before) == []
    res = hostsim.apply_actual()
    assert (res.n_lbs, res.n_accels, res.slab_base, res.slab_len) == (len(actual["lbs"]), len(actual["accelerators"]), 0, int(snap.actual.slab_len))


def test_hostsim_empty_delta_and_delete_everything(garecon, oracle, hostsim):
    objects, actual, snap = _small(garecon, 7)
    hostsim.load(snap)
    before = hostsim.diff()
    model, om = AwsModel(actual, snap), Mirror(objects, snap)
    assert tuple(hostsim.apply_actual()) == model.expected(0)
    assert tuple(hostsim.apply_actual(garecon.pack([], {}).actual)) == model.expected(0)  # rows without LBs, accelerators or zones
    assert hostsim.diff().diff(before) == []
    d = {"lb_deleted": list(range(len(actual["lbs"]))), "acc_deleted": list(range(len(actual["accelerators"])))[::-1],
         "zones": [(z, []) for z in range(len(actual["zones"]))]}
    res = apply_delta(garecon, hostsim, model, d)
    assert res.n_lbs == res.n_accels == res.n_records == res.n_values == 0
    msnap = garecon.pack(om.objects, model.actual)
    assert_same_full(hostsim.diff(), oracle.diff(msnap, "default", mode=1), om.slab, msnap.arrays["o.slab"])


def test_hostsim_delta_before_load_is_a_state_error(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    with garecon.Engine(cluster_name="default", lib=lib) as e:
        with pytest.raises(garecon.GarError) as ei:
            e.apply_actual(lb_deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE


def test_ctypes_actual_delta_struct_sizes_match_header(garecon):
    src = textwrap.dedent('''
        #include <stdio.h>
        #include "garecon.h"
        int main(void) { printf("%zu %zu\\n", sizeof(gar_actual_delta), sizeof(gar_actual_delta_result)); return 0; }
    ''')
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(REPO / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout.split()
    abi = garecon.abi
    assert [int(x) for x in out] == [ctypes.sizeof(abi.GarActualDelta), ctypes.sizeof(abi.GarActualDeltaResult)]


# ------------------------------------------------------------------ table-level churn (deltas.py: what profiles/actual_delta_bench.py runs)

def aws_churn_sequence(garecon, engine, snap, n_batches, seed, max_zones=4):
    """Load `snap`, apply `n_batches` aws_churn batches; checks the results against deltas.ActualMirror.  -> mirror snapshot."""
    deltas, tables = deltas_mod(), garecon.tables
    engine.load(snap)
    m = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    rng = np.random.default_rng(seed)
    for _ in range(n_batches):
        d = deltas.aws_churn(m, rng, max_zones=max_zones)
        keep, rows = deltas.actual_struct(d["rows"])
        res = engine.apply_actual(rows, d["lb_target"], d["acc_target"], d["zone_target"], d["lb_deleted"], d["acc_deleted"])
        want = m.apply(**d)
        assert tuple(res) == tuple(want[k] for k in garecon.abi.ActualDeltaResult.FIELDS)
    return m.snapshot(tables.columns(snap.objects, tables.OBJ_TABLES))


def test_hostsim_table_churn_matches_actual_mirror(garecon, oracle, hostsim):
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, 3000)
    msnap = aws_churn_sequence(garecon, hostsim, snap, 3, 21)
    got = hostsim.diff()
    want = oracle.diff(msnap, snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    rows = list(range(0, int(msnap.objects.n_objects), 97))
    got = hostsim.diff_keys(rows)
    want = oracle.diff_keys(msnap, rows, [], cluster=snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


# ------------------------------------------------------------------ GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(500, 512))
def test_gpu_random_sequences(garecon, oracle, engine, seed):
    run_sequence(garecon, oracle, engine, seed, n_objects=80, n_batches=random.Random(seed).randrange(4, 9), oracle_mode=1)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_gpu_converges_without_reload(garecon, oracle, engine, seed):
    converge(garecon, oracle, engine, seed, 1)


@pytest.mark.gpu
def test_gpu_invalid_and_state_errors(garecon, oracle, engine):
    objects, actual, snap = _small(garecon)
    engine.load(snap)
    before = engine.diff()
    rows = garecon.pack([], {"zones": [actual["zones"][0]]})
    other = next(i for i, x in enumerate(actual["zones"]) if x["name"] != actual["zones"][0]["name"])
    with pytest.raises(garecon.GarError) as ei:
        engine.apply_actual(rows.actual, zone_target=[other])
    assert ei.value.rc == garecon.abi.GAR_E_INVALID
    with pytest.raises(garecon.GarError) as ei:
        engine.apply_actual(acc_deleted=[0, 0])
    assert ei.value.rc == garecon.abi.GAR_E_INVALID
    assert engine.diff().diff(before) == []
    with garecon.Engine(cluster_name="default") as e:
        with pytest.raises(garecon.GarError) as ei:
            e.apply_actual(lb_deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE


@pytest.mark.gpu
def test_gpu_attached_and_sharded_are_state_errors(garecon):
    import torch
    objects, actual, snap = _small(garecon)
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
        with pytest.raises(garecon.GarError) as ei:
            e.apply_actual(lb_deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE
        e.load(snap)
        e.shard_route(garecon.abi.GarShard(0, 1, 0, 0, 0, 0, 0, 0, 0), 1)
        with pytest.raises(garecon.GarError) as ei:
            e.apply_actual(lb_deleted=[0])
        assert ei.value.rc == garecon.abi.GAR_E_STATE


@pytest.mark.gpu
def test_gpu_table_churn_at_scale(garecon, oracle, engine):
    """One aws_churn batch at 10^5 objects (configs[2]): full diff and an incremental diff equal the oracle on the mirrored tables."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, 100_000)
    msnap = aws_churn_sequence(garecon, engine, snap, 1, 31)
    got = engine.diff()
    want = oracle.diff(msnap, snap.cluster, mode=1, threads=8)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    rows = list(range(0, int(msnap.objects.n_objects), 101))
    got = engine.diff_keys(rows)
    want = oracle.diff_keys(msnap, rows, [], cluster=snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


@pytest.mark.gpu
def test_gpu_hot_txt_sets(garecon, oracle, engine):
    """The config-5 shape (hot TXT sets of ~10^5 values): replacing the record lists of every zone keeps parity."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(5, 20_000)
    msnap = aws_churn_sequence(garecon, engine, snap, 1, 33, max_zones=1 << 20)
    got = engine.diff()
    want = oracle.diff(msnap, snap.cluster, mode=1, threads=8)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


@pytest.mark.gpu
def test_gpu_launch_count_after_aws_delta(garecon):
    """The first full diff after an AWS delta prepares the snapshot exactly as the first one after a load (same launches), and
    later full diffs record and replay the launch sequence as after a load."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    deltas = deltas_mod()
    snap = synth.generate(3, 20_000)
    with garecon.Engine(cluster_name=snap.cluster) as e:
        e.load(snap)
        e.diff_raw()  # capacities settle on the first snapshot of this shape: later loads start with buffers that fit
        e.load(snap)
        after_load = [e.diff_raw()["kernel_launches"] for _ in range(4)]
        m = deltas.ActualMirror(garecon.tables.columns(snap.actual, garecon.tables.ACT_TABLES))
        d = deltas.aws_churn(m, np.random.default_rng(41))
        keep, rows = deltas.actual_struct(d["rows"])
        e.apply_actual(rows, d["lb_target"], d["acc_target"], d["zone_target"], d["lb_deleted"], d["acc_deleted"])
        after_delta = [e.diff_raw()["kernel_launches"] for _ in range(4)]
    assert after_delta == after_load, (after_delta, after_load)
