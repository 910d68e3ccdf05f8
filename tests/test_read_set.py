"""gar_read_set: the resident AWS rows the decisions of a keyset read.

Exactness against the Python restatement of the rules (tests/readset_ref.py, built on oracle/pyref.py's helpers), sufficiency
(every row outside the set rewritten in the columns that do not decide membership leaves gar_diff_keys' answer unchanged), the
stale-mirror scenarios the call exists for, and its interplay with the prepared state.  The cases run on the host simulation
(CPU tier) and on the GPU."""
import copy
import random

import numpy as np
import pytest

import hotkeys
import multilbi
import randmodel
import readset_ref
import scalemodels

from oracle import pyref

OBJ, ACT = 1, 2


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


_alive = {}


def load(garecon, e, objects, actual):
    """Load a packed snapshot; the host simulation reads the caller's columns in place, so they stay alive until the next load."""
    snap = garecon.pack(objects, actual)
    e.load(snap)
    _alive[id(e)] = [snap]
    return snap


def slab_str(e, ref):
    ref = int(ref)
    return bytes(e.read_slab(OBJ, ref & ((1 << 40) - 1), ref >> 40)).decode()


def got(e, rows, deleted=()):
    rs = e.read_set(rows, deleted)
    for k in ("lb_rows", "acc_rows", "zone_rows"):
        a = getattr(rs, k)
        assert np.all(a[1:] > a[:-1]), k  # ascending, distinct
    misses = [(int(o), int(j), slab_str(e, n), slab_str(e, r)) for o, j, n, r in zip(rs.lb_miss_obj, rs.lb_miss_j, rs.lb_miss_name, rs.lb_miss_region)]
    assert misses == sorted(misses)
    return {"lbs": rs.lb_rows.tolist(), "accs": rs.acc_rows.tolist(), "zones": rs.zone_rows.tolist(), "misses": misses}


def want(objects, actual, rows, deleted=()):
    return readset_ref.read_set(objects, copy.deepcopy(actual), "default", rows, deleted)


def keysets(objects, actual, rng, deleted_pool):
    n = len(objects)
    sets = [[], [rng.randrange(n)], rng.sample(range(n), max(1, n // 100)), rng.sample(range(n), max(1, n // 10)), list(range(n))]
    sets.append([rng.randrange(n) for _ in range(20)] * 2)  # duplicate rows
    out = [(s, []) for s in sets]
    out.append((sets[2], deleted_pool))
    out.append(([], deleted_pool))
    return out


def deleted_keys(objects, actual, extra=()):
    """Keys whose objects are gone but whose resources remain, keys that own nothing, and keys that are not "ns/name"."""
    return list(extra) + scalemodels.ABSENT_KEYS


def check_model(garecon, e, objects, actual, seed, deleted=()):
    load(garecon, e, objects, actual)
    rng = random.Random(seed)
    for rows, dk in keysets(objects, actual, rng, deleted_keys(objects, actual, deleted)):
        assert got(e, rows, dk) == want(objects, actual, rows, dk), (len(rows), len(dk))


@pytest.mark.parametrize("seed", range(8))
def test_exact_randmodel(garecon, eng, seed):
    objects, actual = randmodel.make(seed, n_objects=60)
    check_model(garecon, eng, objects, actual, seed)


@pytest.mark.parametrize("seed", range(3))
def test_exact_randmodel_dropped(garecon, eng, seed):
    objects, actual, dropped = scalemodels.randmodel_dropped(seed, 400)
    check_model(garecon, eng, objects, actual, seed, dropped)


@pytest.mark.parametrize("seed", range(3))
def test_exact_multilbi(garecon, eng, seed):
    objects, actual = multilbi.make(seed, n_objects=50)
    check_model(garecon, eng, objects, actual, seed)


def test_exact_hotkeys(garecon, eng):
    objects, actual = hotkeys.make()
    check_model(garecon, eng, objects, actual, 5, [scalemodels.key_of(ob) for ob in objects[:3]])
    objects, actual = scalemodels.hot_cluster(2, 300)
    check_model(garecon, eng, objects, actual, 6)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(2))
def test_exact_gpu_scale(garecon, engine, seed):
    objects, actual, dropped = scalemodels.randmodel_dropped(seed, 20000)
    check_model(garecon, engine, objects, actual, seed, dropped[:100])
    objects, actual = scalemodels.hot_cluster(seed, 20000)
    check_model(garecon, engine, objects, actual, seed)


# ---------------------------------------------------------------- sufficiency

def rewrite_outside(actual, rs, keys, rng):
    """An AWS delta that replaces every LB, accelerator subtree and zone record list outside the read set, keeping the columns
    that decide membership (LB region / name, accelerator tags, zone name) and giving zones records with no owner value of a key.
    Child counts (listeners, endpoint groups per listener, records, values per record) are kept, so that the child rows the ops
    name keep their numbers and the change set must stay identical."""
    lbs = [(r, dict(lb, dns=f"x{r}.elb.amazonaws.com", arn=f"arn:new:{r}", state=rng.choice(["active", "provisioning", "failed"])))
           for r, lb in enumerate(actual["lbs"]) if r not in set(rs["lbs"])]
    accs = []
    for r, a in enumerate(actual["accelerators"]):
        if r in set(rs["accs"]):
            continue
        lis = [{"proto": rng.choice(["TCP", "UDP"]), "ports": [rng.randrange(1, 9000) for _ in range(rng.randrange(0, 3))],
                "egs": [{"endpoints": [f"arn:ep:{rng.randrange(99)}" for _ in range(rng.randrange(0, 3))]} for _ in li.get("egs", [])]}
               for li in a.get("listeners", [])]
        accs.append((r, dict(a, name=f"n{r}", dns=f"d{r}.awsglobalaccelerator.com", enabled=not a.get("enabled", True), listeners=lis)))
    zones = []
    for r, z in enumerate(actual["zones"]):
        if r in set(rs["zones"]):
            continue
        recs = []
        for k, rec in enumerate(z.get("records", [])):
            nr = {"name": f"r{k}.{z['name']}", "type": rng.choice(["A", "TXT"]), "values": [f'"v{k}.{x}"' for x in range(len(rec.get("values", [])))]}
            if rng.random() < 0.3:
                nr["alias"] = f"z{r}.awsglobalaccelerator.com."
            recs.append(nr)
        zones.append((r, recs))
    return {"lbs": lbs, "accs": accs, "zones": zones}


def apply_rows(garecon, e, actual, d):
    rows = {"lbs": [x for _, x in d["lbs"]], "accelerators": [x for _, x in d["accs"]],
            "zones": [dict(actual["zones"][z], records=r) for z, r in d["zones"]]}
    packed = garecon.pack([], rows)
    _alive.setdefault(id(e), []).append(packed)
    e.apply_actual(packed.actual, [t for t, _ in d["lbs"]], [t for t, _ in d["accs"]], [z for z, _ in d["zones"]])


def check_sufficiency(garecon, e, objects, actual, seed, deleted):
    rng = random.Random(seed)
    n = len(objects)
    rows = rng.sample(range(n), max(1, n // rng.choice([2, 10, 50])))
    dk = rng.sample(deleted, min(len(deleted), 5)) + [(0, "default/absent")]
    load(garecon, e, objects, actual)
    before = e.diff_keys(rows, dk)
    rs = got(e, rows, dk)
    apply_rows(garecon, e, actual, rewrite_outside(actual, rs, dk, rng))
    after = e.diff_keys(rows, dk)
    assert after.diff(before) == [], after.describe_first_mismatch(before)


@pytest.mark.parametrize("seed", range(12))
def test_sufficiency(garecon, hostsim, seed):
    objects, actual, dropped = scalemodels.randmodel_dropped(seed, 120)
    check_sufficiency(garecon, hostsim, objects, actual, seed, dropped)


@pytest.mark.parametrize("seed", range(2))
def test_sufficiency_multilbi_hot(garecon, hostsim, seed):
    check_sufficiency(garecon, hostsim, *multilbi.make(seed, n_objects=60), seed, [])
    objects, actual = scalemodels.hot_cluster(seed, 200)
    check_sufficiency(garecon, hostsim, objects, actual, seed, [scalemodels.key_of(ob) for ob in objects[:4]])


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_sufficiency_gpu(garecon, engine, seed):
    objects, actual, dropped = scalemodels.randmodel_dropped(seed, 5000)
    check_sufficiency(garecon, engine, objects, actual, seed, dropped)


# ---------------------------------------------------------------- the stale mirror the call exists for

def managed_rows(objects, actual, e, garecon):
    """Rows whose GA decision reaches an active load balancer (status OK) in `actual`, with their first lbIngress LB row."""
    load(garecon, e, objects, actual)
    rows = list(range(len(objects)))
    cs = e.diff_keys(rows)
    out = []
    for k, i in enumerate(rows):
        if (int(cs.status_ga[k]) & 0xFF) == pyref.ST_OK and int(cs.derived[k]) & 32 and objects[i].get("lb_ingress"):  # GAR_DV_GA_MANAGED
            code, name, region = pyref.tokenise(objects[i]["lb_ingress"][0])
            lbs = [r for r, lb in enumerate(actual["lbs"]) if (lb["region"], lb["name"]) == (region, name)]
            if code <= 2 and len(lbs) == 1 and len(objects[i]["lb_ingress"]) == 1:
                out.append((i, lbs[0]))
    return out


def refresh(garecon, e, cloud, rows, deleted=()):
    """The worker loop: read set -> re-describe those rows from the cloud tables -> one AWS delta."""
    rs = got(e, rows, deleted)
    d = {"lbs": [(r, cloud["lbs"][r]) for r in rs["lbs"]], "accs": [(r, cloud["accelerators"][r]) for r in rs["accs"]],
         "zones": [(z, cloud["zones"][z]["records"]) for z in rs["zones"]]}
    apply_rows(garecon, e, cloud, d)
    return rs


def test_stale_provisioning_lb(garecon, oracle, eng):
    objects, cloud = randmodel.make(3, n_objects=80)
    i, lb = managed_rows(objects, cloud, eng, garecon)[0]
    stale = copy.deepcopy(cloud)
    stale["lbs"][lb]["state"] = "provisioning"
    load(garecon, eng, objects, stale)
    assert (int(eng.diff_keys([i]).status_ga[0]) & 0xFF) == pyref.ST_REQUEUE_30S  # the hole: every requeue sees the same row
    refresh(garecon, eng, cloud, [i])
    want_cs = oracle.diff_keys(garecon.pack(objects, cloud), [i], mode=0)
    assert eng.diff_keys([i]).diff(want_cs) == []


def test_stale_missing_lb(garecon, oracle, eng):
    objects, cloud = randmodel.make(4, n_objects=80)
    i, lb = managed_rows(objects, cloud, eng, garecon)[0]
    stale = copy.deepcopy(cloud)
    gone = stale["lbs"].pop(lb)
    load(garecon, eng, objects, stale)
    assert (int(eng.diff_keys([i]).status_ga[0]) >> 8 & 0xFF) == 5  # GAR_D_LB_NOT_FOUND
    rs = got(eng, [i])
    assert (i, 0, gone["name"], gone["region"]) in rs["misses"]
    # the worker describes the missing load balancer by (region, name) and appends it
    packed = garecon.pack([], {"lbs": [gone], "accelerators": [], "zones": []})
    _alive[id(eng)].append(packed)
    eng.apply_actual(packed.actual, [0xFFFFFFFF], [], [])
    now = copy.deepcopy(stale)
    now["lbs"].append(gone)
    assert eng.diff_keys([i]).diff(oracle.diff_keys(garecon.pack(objects, now), [i], mode=0)) == []


def test_stale_drift_and_deleted_record(garecon, oracle, eng):
    """Port / endpoint drift on owned accelerators and owned records deleted out of band reach the keys through the refresh."""
    objects, stale = randmodel.make(5, n_objects=80)
    cloud = copy.deepcopy(stale)
    for a in cloud["accelerators"]:
        for li in a.get("listeners", []):
            li["ports"] = [p + 1 for p in li.get("ports", [])]
            for eg in li.get("egs", []):
                eg["endpoints"] = eg.get("endpoints", [])[1:]
    for z in cloud["zones"]:
        z["records"] = [r for r in z.get("records", []) if r.get("alias") is None]
    rows = list(range(len(objects)))
    load(garecon, eng, objects, stale)
    stale_cs = eng.diff_keys(rows)
    want_cs = oracle.diff_keys(garecon.pack(objects, cloud), rows, mode=0)
    assert stale_cs.diff(want_cs) != []  # the stale mirror answers from rows that are gone
    refresh(garecon, eng, cloud, rows)
    assert eng.diff_keys(rows).diff(want_cs) == []


def test_stale_deleted_key_accelerator_gone(garecon, oracle, eng):
    objects, actual, dropped = scalemodels.randmodel_dropped(6, 300)
    load(garecon, eng, objects, actual)
    owning = [k for k in dropped if got(eng, [], [k])["accs"]]
    key = owning[0]
    rs = got(eng, [], [key])
    cloud = copy.deepcopy(actual)
    eng.apply_actual(None, [], [], [], [], rs["accs"])  # the accelerators are already gone in the cloud
    for r in sorted(rs["accs"], reverse=True):
        cloud["accelerators"].pop(r)
    cs = eng.diff_keys([], [key])
    assert not any((int(op[0]) & 0xFF) == 7 for op in cs.ops.tolist())  # no GA_DELETE_CHAIN for it
    assert cs.diff(oracle.diff_keys(garecon.pack(objects, cloud), [], [key], mode=0)) == []


# ---------------------------------------------------------------- interplay and edges

def export_bytes(e):
    x = e.export(OBJ | ACT)
    return x.buf.tobytes()


def test_nothing_resident_changes_and_replay(garecon, eng):
    objects, actual, dropped = scalemodels.randmodel_dropped(7, 300)
    load(garecon, eng, objects, actual)
    for _ in range(4):  # load, first diff on the prepared snapshot, recording, replay
        eng.diff()
    mode = eng.counters()["launch_mode"]
    before = export_bytes(eng)
    rows = list(range(0, len(objects), 7))
    first = got(eng, rows, dropped[:5])
    assert got(eng, rows, dropped[:5]) == first
    assert export_bytes(eng) == before
    eng.diff()
    assert eng.counters()["launch_mode"] == mode  # 2 on the GPU: the recorded diff still replays
    # after deltas and compactions the call prepares as gar_diff_keys does
    up = garecon.pack(objects[:5], None)
    _alive[id(eng)].append(up)
    eng.apply_objects(up.objects, [scalemodels.key_of(objects[-1])])
    eng.compact(OBJ | ACT)
    eng.apply_zones(None, [], [0])
    x = eng.export(OBJ | ACT)
    rows = list(range(0, int(x.objects.n_objects), 5))
    a = got(eng, rows, dropped[:5])
    eng.load(x)
    _alive[id(eng)] = [x]
    assert got(eng, rows, dropped[:5]) == a  # the same tables freshly loaded give the same set


def test_edges(garecon, eng):
    with garecon.Engine(cluster_name="default", lib=eng.lib) as fresh:
        with pytest.raises(garecon.abi.GarError) as ei:
            fresh.read_set([0])
    assert ei.value.rc == -4  # GAR_E_STATE before a load
    objects, actual = randmodel.make(8, n_objects=70)
    load(garecon, eng, objects, actual)
    assert got(eng, []) == {"lbs": [], "accs": [], "zones": [], "misses": []}
    for bad in ([len(objects)], [0, 1 << 31]):
        with pytest.raises(garecon.abi.GarError) as ei:
            eng.read_set(bad)
        assert ei.value.rc == -1
    with pytest.raises(garecon.abi.GarError):
        eng.read_set([0], [(2, "ns/x")])
    rows = [0, 31, 32, 63, 64, len(objects) - 1]
    assert got(eng, rows) == want(objects, actual, rows)
    # tables of 2^k +- 1 rows: bitmap word boundaries in every section
    for n in (31, 33, 63, 65):
        o, a = randmodel.make(n, n_objects=n)
        a["lbs"] = (a["lbs"] * 3)[:n]
        load(garecon, eng, o, a)
        assert got(eng, list(range(n))) == want(o, a, list(range(n)))
    # empty AWS tables: everything misses
    load(garecon, eng, objects, {"lbs": [], "accelerators": [], "zones": []})
    r = got(eng, list(range(len(objects))))
    assert r == want(objects, {"lbs": [], "accelerators": [], "zones": []}, list(range(len(objects))))
    assert r["lbs"] == r["accs"] == r["zones"] == []


def test_tiny_caps_and_no_graph(garecon, monkeypatch):
    import __graft_entry__ as ge
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    monkeypatch.setenv("GAR_NO_GRAPH", "1")
    lib = garecon.abi.load_library(ge.build_hostsim())
    with garecon.Engine(cluster_name="default", lib=lib) as e:
        objects, actual = multilbi.make(9, n_objects=60)
        check_model(garecon, e, objects, actual, 9)


@pytest.mark.gpu
def test_tiny_caps_and_no_graph_gpu(garecon, monkeypatch):
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    monkeypatch.setenv("GAR_NO_GRAPH", "1")
    with garecon.Engine(cluster_name="default", device=0) as e:
        objects, actual = multilbi.make(9, n_objects=60)
        check_model(garecon, e, objects, actual, 9)
        e.diff()
        e.diff()
        assert e.counters()["launch_mode"] == 0


@pytest.mark.gpu
def test_no_skew_cliff(garecon, engine):
    """One key owning 10^5 accelerators and 10^5 owner values: its read set takes at most 5x (plus 1 ms) the time of a key owning
    one of each, because every owned row is its own item of the marking pass."""
    import time
    n = 100_000
    hot = {"kind": "service", "ns": "default", "name": "hot", "lb_ingress": [], "annotations": {}}
    cold = {"kind": "service", "ns": "default", "name": "cold", "lb_ingress": [], "annotations": {}}
    tags = lambda key: [("aws-global-accelerator-controller-managed", "true"), ("aws-global-accelerator-owner", f"service/default/{key}"),
                        ("aws-global-accelerator-cluster", "default")]
    val = lambda key: f'"heritage=aws-global-accelerator-controller,cluster=default,service/default/{key}"'
    accs = [{"name": f"a{k}", "dns": f"a{k}.x", "tags": tags("hot"), "listeners": []} for k in range(n)]
    accs.append({"name": "c", "dns": "c.x", "tags": tags("cold"), "listeners": []})
    recs = [{"name": f"r{k}.example.com.", "type": "TXT", "values": [val("hot")]} for k in range(n)]
    recs.append({"name": "c.example.com.", "type": "TXT", "values": [val("cold")]})
    actual = {"lbs": [], "accelerators": accs, "zones": [{"name": "example.com.", "records": recs}]}
    load(garecon, engine, [hot, cold], actual)

    def timed(rows):
        ts = []
        for _ in range(7):
            t0 = time.perf_counter()
            rs = engine.read_set(rows)
            ts.append(time.perf_counter() - t0)
        return sorted(ts)[3], rs
    timed([1])
    t_cold, rs_cold = timed([1])
    t_hot, rs_hot = timed([0])
    assert rs_hot.acc_rows.size == n and rs_cold.acc_rows.tolist() == [n]
    assert t_hot <= 5 * t_cold + 1e-3, (t_hot, t_cold)
