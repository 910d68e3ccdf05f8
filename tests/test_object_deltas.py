"""Object deltas (gar_snapshot_apply_objects): informer events applied to the resident object table.  After every batch the
engine must answer exactly as a fresh gar_snapshot_load of the table a small Python mirror of the rules holds (include/
garecon.h "object deltas"): full diff, incremental diff of the touched keys and the EndpointGroupBinding set-diff, all
against the oracle.  tok_name / tok_region point into the resident slab (loaded bytes, then each delta's strings at its
slab_base) and are compared as the strings they name; every other array bit for bit."""
import copy
import ctypes
import random
import subprocess
import tempfile
import textwrap
from pathlib import Path

import numpy as np
import pytest

import egbcases
import randmodel

REPO = Path(__file__).resolve().parent.parent
NONE = 0xFFFFFFFF
ANN = randmodel.ANN


def key_of(ob):
    return (0 if ob.get("kind", "service") == "service" else 1, f"{ob.get('ns', 'default')}/{ob['name']}")


class Mirror:
    """The rules of include/garecon.h on a list of objects (the dict model of tables.pack), plus the resident slab."""

    def __init__(self, objects, snap):
        self.objects = list(objects)
        self.slab = bytearray(snap.arrays["o.slab"][:int(snap.objects.slab_len)].tobytes())

    def _lowest(self, k):
        return next((i for i, ob in enumerate(self.objects) if key_of(ob) == k), NONE)

    def apply(self, upserts, deleted, upsert_snap=None):
        deleted_row, moved_from, upsert_row = [], [], []
        for k in deleted:
            r = self._lowest(k)
            deleted_row.append(r)
            moved_from.append(NONE if r in (NONE, len(self.objects) - 1) else len(self.objects) - 1)
            if r != NONE:
                self.objects[r] = self.objects[-1]
                self.objects.pop()
        for ob in upserts:
            r = self._lowest(key_of(ob))
            if r == NONE:
                r = len(self.objects)
                self.objects.append(ob)
            else:
                self.objects[r] = ob
            upsert_row.append(r)
        base = 0
        if upserts:
            base = (len(self.slab) + 15) & ~15
            self.slab += b"\0" * (base - len(self.slab))
            self.slab += upsert_snap.arrays["o.slab"][:int(upsert_snap.objects.slab_len)].tobytes()
        return upsert_row, deleted_row, moved_from, base


def _strings(refs, slab):
    return [bytes(slab[int(r) & ((1 << 40) - 1):(int(r) & ((1 << 40) - 1)) + (int(r) >> 40)]) for r in refs]


def assert_same_full(got, want, got_slab, want_slab):
    for k in got.ARRAYS:
        a, b = getattr(got, k), getattr(want, k)
        if k in ("tok_name", "tok_region"):
            assert _strings(a, got_slab) == _strings(b, want_slab), k
        else:
            assert a.shape == b.shape and np.array_equal(a, b), f"{k}: {got.describe_first_mismatch(want)}"


class Events:
    """Random informer events over a randmodel cluster: in-place updates (annotations, lbIngress hostnames, ports, spec type,
    class), adds (fresh keys, and keys that own existing accelerators or records), deletes (keys that own resources) and
    keys that are not in the cache."""

    def __init__(self, seed, actual):
        self.rng = random.Random(seed * 31 + 5)
        self.pool = randmodel.make(seed + 9000, n_objects=30)[0]
        owners = [dict(a["tags"]).get("aws-global-accelerator-owner", "") for a in actual.get("accelerators", [])]
        for z in actual.get("zones", []):
            for r in z.get("records", []):
                owners += [v.rsplit(",", 1)[1].rstrip('"') for v in r.get("values", []) if v.startswith('"heritage=') and v.count(",") >= 2]
        self.owner_keys = sorted({(0 if p[0] == "service" else 1, f"{p[1]}/{p[2]}") for p in (o.split("/") for o in owners)
                                  if len(p) == 3 and p[0] in ("service", "ingress")})
        self.serial = 0

    def _update(self, ob, objects):
        rng = self.rng
        ob = copy.deepcopy(ob)
        ann = ob.setdefault("annotations", {})
        for _ in range(rng.randrange(1, 4)):
            c = rng.randrange(7)
            if c == 0:
                other = rng.choice(objects)
                ob["lb_ingress"] = list(other.get("lb_ingress", [])) if rng.random() < 0.7 else rng.choice([[], ["example.com"], ["a.b"]])
            elif c == 1:
                src = rng.choice(objects).get("annotations", {})
                v = src.get(ANN + "route53-hostname") if isinstance(src, dict) else None
                if v is None or rng.random() < 0.3:
                    ann.pop(ANN + "route53-hostname", None)
                else:
                    ann[ANN + "route53-hostname"] = v
            elif c == 2:
                if ann.pop(ANN + "global-accelerator-managed", None) is None:
                    ann[ANN + "global-accelerator-managed"] = "true"
            elif c == 3:
                if ob.get("kind") == "service":
                    ob["ports"] = [(rng.choice([80, 443, 53, 8443]), rng.choice(["TCP", "UDP"])) for _ in range(rng.randrange(0, 4))]
                else:
                    ob["ports"] = [rng.choice([80, 443, 0]) for _ in range(rng.randrange(0, 3))]
            elif c == 4:
                if ob.get("kind") == "service":
                    ob["spec_type"] = rng.choice(["LoadBalancer", "LoadBalancer", "ClusterIP", "NodePort"])
                else:
                    ob["ingress_class"] = rng.choice(["alb", "nginx", None])
            elif c == 5:
                ann["alb.ingress.kubernetes.io/listen-ports"] = rng.choice(randmodel.LISTEN_PORTS)
            else:
                ann[ANN + "global-accelerator-name"] = rng.choice(["custom-name", "", f"n{rng.randrange(100)}"])
        return ob

    def batch(self, objects):
        rng = self.rng
        used, deleted, upserts = set(), [], []
        present = {key_of(o) for o in objects}

        def take(k):
            if k in used:
                return False
            used.add(k)
            return True

        for _ in range(rng.randrange(0, 5)):  # deletes: objects in the cache (most own accelerators / records), and absent keys
            k = key_of(rng.choice(objects)) if objects and rng.random() < 0.8 else (rng.randrange(2), f"default/absent-{rng.randrange(50)}")
            if take(k):
                deleted.append(k)
        for _ in range(rng.randrange(0, 6)):  # in-place updates
            if objects:
                ob = self._update(rng.choice(objects), objects)
                if take(key_of(ob)):
                    upserts.append(ob)
        for _ in range(rng.randrange(0, 3)):  # adds with fresh keys
            self.serial += 1
            ob = copy.deepcopy(rng.choice(self.pool))
            ob["name"] = f"add{self.serial}-{ob['name']}"
            if take(key_of(ob)):
                upserts.append(ob)
        absent_owners = [k for k in self.owner_keys if k not in present]
        for k in rng.sample(absent_owners, min(len(absent_owners), rng.randrange(0, 3))):  # adds that adopt orphaned resources
            kind_name = "service" if k[0] == 0 else "ingress"
            base = [o for o in self.pool if o.get("kind", "service") == kind_name]
            if not base:
                continue
            ob = copy.deepcopy(rng.choice(base))
            ob["ns"], ob["name"] = k[1].split("/", 1)
            if take(key_of(ob)):
                upserts.append(ob)
        rng.shuffle(upserts)
        return upserts, deleted


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


def run_sequence(garecon, oracle, engine, seed, n_objects, n_batches, oracle_mode, check_keys=True, check_bindings=True):
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=n_objects, n_bindings=3 * n_objects)
    snap = garecon.pack(objects, actual)
    b = garecon.pack_bindings(bindings, known)
    engine.load(snap)
    mirror = Mirror(objects, snap)
    events = Events(seed, actual)
    if seed % 3 == 0:
        engine.diff()  # a prepared snapshot (digests + indexes resident) for some sequences, a fresh one for the others
    for _ in range(n_batches):
        upserts, deleted = events.batch(mirror.objects)
        usnap = garecon.pack(upserts, None) if upserts else None
        res = engine.apply_objects(usnap.objects if usnap else None, deleted)
        up_row, del_row, moved, base = mirror.apply(upserts, deleted, usnap)
        assert res.upsert_row.tolist() == up_row
        assert res.deleted_row.tolist() == del_row
        assert res.moved_from.tolist() == moved
        assert res.n_objects == len(mirror.objects)
        assert res.slab_len == len(mirror.slab)
        if upserts:
            assert res.slab_base == base
        msnap = garecon.pack(mirror.objects, actual)
        if check_keys:
            got = engine.diff_keys(up_row, deleted)
            want = oracle.diff_keys(msnap, up_row, deleted, mode=oracle_mode)
            assert got.diff(want) == [], got.describe_first_mismatch(want)
        got = engine.diff()
        want = oracle.diff(msnap, "default", mode=1)
        assert_same_full(got, want, mirror.slab, msnap.arrays["o.slab"])
        if check_bindings:
            assert engine.bindings_diff(b).ops.tolist() == oracle.bindings_diff(msnap, b).ops.tolist()
    return mirror


@pytest.mark.parametrize("seed", range(20))
def test_hostsim_random_sequences(garecon, oracle, hostsim, seed):
    rng = random.Random(seed)
    run_sequence(garecon, oracle, hostsim, seed, n_objects=30, n_batches=rng.randrange(5, 11), oracle_mode=0)


def test_hostsim_sequence_with_tiny_capacities(garecon, oracle, hostsim, monkeypatch):
    """Every capacity starts at 1: the regrow-and-rerun paths of the diff run on a table that deltas changed."""
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    run_sequence(garecon, oracle, hostsim, 101, n_objects=30, n_batches=6, oracle_mode=0)


def test_hostsim_empty_delta_is_a_no_op(garecon, oracle, hostsim):
    objects, actual = randmodel.make(3, n_objects=20)
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    before = hostsim.diff()
    res = hostsim.apply_objects(None, [])
    assert (res.n_objects, res.slab_base, res.slab_len) == (20, 0, int(snap.objects.slab_len))
    assert hostsim.diff().diff(before) == []
    res = hostsim.apply_objects(None, [(0, "default/never-existed"), (1, "no-slash")])
    assert res.deleted_row.tolist() == [NONE, NONE] and res.moved_from.tolist() == [NONE, NONE]
    assert hostsim.diff().diff(before) == []


def test_hostsim_delete_everything(garecon, oracle):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    objects, actual = randmodel.make(4, n_objects=12)
    snap = garecon.pack(objects, actual)
    keys = [key_of(o) for o in objects]
    with garecon.Engine(cluster_name="default", lib=lib) as e:
        e.load(snap)
        m = Mirror(objects, snap)
        order = list(keys)
        random.Random(4).shuffle(order)
        res = e.apply_objects(None, order)
        _, del_row, moved, _ = m.apply([], order)
        assert res.deleted_row.tolist() == del_row and res.moved_from.tolist() == moved and res.n_objects == 0
        with pytest.raises(garecon.GarError) as ei:
            e.diff()
        assert ei.value.rc == garecon.abi.GAR_E_STATE
    with garecon.Engine(cluster_name="default", lib=lib, allow_empty_cache=True) as e:
        e.load(snap)
        e.apply_objects(None, order)
        got = e.diff()
        want = oracle.diff(garecon.pack([], actual), "default", mode=1)
        assert got.diff(want) == [], got.describe_first_mismatch(want)


def _two_upserts(garecon):
    obs = [dict(kind="service", ns="default", name="u-one", spec_type="LoadBalancer", annotations={"a": "b", ANN + "global-accelerator-managed": "true"},
                lb_ingress=["x-0123456789abcdef.elb.us-east-1.amazonaws.com"], ports=[(80, "TCP")]),
           dict(kind="ingress", ns="prod", name="u-two", ingress_class="alb", annotations={"c": "d"}, lb_ingress=[], ports=[80, 443])]
    return garecon.pack(obs, None)


@pytest.mark.parametrize("breakage", ["csr", "string", "kind", "layout", "twice", "delete_and_upsert"])
def test_hostsim_invalid_delta_changes_nothing(garecon, oracle, hostsim, breakage):
    objects, actual = randmodel.make(5, n_objects=20)
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    before = hostsim.diff()
    u = _two_upserts(garecon)
    deleted = [key_of(objects[3])]
    if breakage == "csr":
        u.arrays["obj_port_begin"][1:] = [3, 2]  # 0, 3, 2: not monotone
    elif breakage == "string":
        u.arrays["ann_val"][0] = (4 << 40) | int(u.objects.slab_len)
    elif breakage == "kind":
        u.arrays["obj_kind"][1] = 2
    elif breakage == "layout":
        u.arrays["obj_name"][0] += 1
    elif breakage == "twice":
        deleted = deleted + deleted
    else:
        deleted = deleted + [(0, "default/u-one")]
    with pytest.raises(garecon.GarError) as ei:
        hostsim.apply_objects(u.objects, deleted)
    assert ei.value.rc == garecon.abi.GAR_E_INVALID
    assert hostsim.diff().diff(before) == []
    res = hostsim.apply_objects(None, [])
    assert res.n_objects == 20 and res.slab_len == int(snap.objects.slab_len)


def test_hostsim_duplicate_keys_follow_the_lowest_row(garecon, oracle, hostsim):
    objects, actual = randmodel.make(6, n_objects=16)
    dup = copy.deepcopy(objects[2])
    dup["lb_ingress"] = []
    objects = objects[:9] + [dup] + objects[9:] + [copy.deepcopy(objects[2])]  # the key of row 2 also at rows 9 and 17
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    m = Mirror(objects, snap)
    k = key_of(objects[2])
    for upserts, deleted in (([], [key_of(objects[0]), k]), ([], [k]), ([copy.deepcopy(objects[5]) | {"ns": k[1].split("/")[0], "name": k[1].split("/")[1]}], []),
                             ([], [k]), ([], [k])):
        usnap = garecon.pack(upserts, None) if upserts else None
        res = hostsim.apply_objects(usnap.objects if usnap else None, deleted)
        up_row, del_row, moved, _ = m.apply(upserts, deleted, usnap)
        assert (res.upsert_row.tolist(), res.deleted_row.tolist(), res.moved_from.tolist()) == (up_row, del_row, moved)
        msnap = garecon.pack(m.objects, actual)
        assert_same_full(hostsim.diff(), oracle.diff(msnap, "default", mode=1), m.slab, msnap.arrays["o.slab"])


def test_hostsim_delta_before_load_is_a_state_error(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    with garecon.Engine(cluster_name="default", lib=lib) as e:
        with pytest.raises(garecon.GarError) as ei:
            e.apply_objects(None, [(0, "default/x")])
        assert ei.value.rc == garecon.abi.GAR_E_STATE


def test_ctypes_delta_struct_sizes_match_header(garecon):
    src = textwrap.dedent('''
        #include <stdio.h>
        #include "garecon.h"
        int main(void) { printf("%zu %zu\\n", sizeof(gar_object_delta), sizeof(gar_delta_result)); return 0; }
    ''')
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(REPO / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout.split()
    abi = garecon.abi
    assert [int(x) for x in out] == [ctypes.sizeof(abi.GarObjectDelta), ctypes.sizeof(abi.GarDeltaResult)]


# ------------------------------------------------------------------ GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(400, 412))
def test_gpu_random_sequences(garecon, oracle, engine, seed):
    rng = random.Random(seed)
    run_sequence(garecon, oracle, engine, seed, n_objects=80, n_batches=rng.randrange(5, 11), oracle_mode=1)


# ------------------------------------------------------------------ table-level churn (deltas.py: what profiles/delta_bench.py runs)

def churn_sequence(garecon, engine, snap, n_batches, seed):
    """Load `snap`, apply `n_batches` 1 % churn batches; checks rows and slab placement against deltas.ColumnMirror.
    -> (mirror snapshot, last batch's upsert rows, last batch's deleted keys)."""
    import importlib
    deltas = importlib.import_module("aws-global-accelerator-controller_b200.deltas")
    tables = garecon.tables
    engine.load(snap)
    m = deltas.ColumnMirror(tables.columns(snap.objects, tables.OBJ_TABLES))
    rng = np.random.default_rng(seed)
    for b in range(n_batches):
        up, deleted = deltas.churn(m, rng, serial=b)
        keep, uobj = deltas.objects_struct(up)
        res = engine.apply_objects(uobj, deleted)
        up_row, del_row, moved = m.apply(up, deleted)
        assert np.array_equal(res.upsert_row, up_row) and np.array_equal(res.deleted_row, del_row) and np.array_equal(res.moved_from, moved)
        assert res.n_objects == len(m.keys) and res.slab_len == m.slab_len
    a_cols = tables.columns(snap.actual, tables.ACT_TABLES)
    return m.snapshot(a_cols), up_row, deleted


def test_hostsim_table_churn_matches_column_mirror(garecon, oracle, hostsim):
    import importlib
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, 3000)
    msnap, rows, deleted = churn_sequence(garecon, hostsim, snap, 3, 11)
    got = hostsim.diff()
    want = oracle.diff(msnap, snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)  # the mirror's slab is the resident one: tok refs match bit for bit
    got = hostsim.diff_keys(rows.tolist(), deleted)
    want = oracle.diff_keys(msnap, rows.tolist(), deleted, cluster=snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


@pytest.mark.gpu
def test_gpu_table_churn_at_scale(garecon, oracle, engine):
    """The snapshot test_gpu_keys_at_scale uses (10^5 objects), three 1 % churn batches: full diff and the last batch's
    incremental diff equal the oracle on the table a reload would need."""
    import importlib
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, 100_000)
    msnap, rows, deleted = churn_sequence(garecon, engine, snap, 3, 12)
    got = engine.diff()
    want = oracle.diff(msnap, snap.cluster, mode=1, threads=8)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    got = engine.diff_keys(rows.tolist(), deleted)
    want = oracle.diff_keys(msnap, rows.tolist(), deleted, cluster=snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


@pytest.mark.gpu
def test_gpu_actual_side_stays_prepared(garecon):
    """After a delta the first diff rebuilds the object side only: no accelerator digests, LB hashes or record preparation."""
    import importlib
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    deltas = importlib.import_module("aws-global-accelerator-controller_b200.deltas")
    snap = synth.generate(3, 20_000)
    actual_side = {"digest_accelerators", "hash_load_balancers", "prepare_records"}
    with garecon.Engine(cluster_name=snap.cluster, stage_timing=True) as e:
        e.load(snap)
        e.diff()
        assert actual_side <= {s[0] for s in e.stage_timings()}
        m = deltas.ColumnMirror(garecon.tables.columns(snap.objects, garecon.tables.OBJ_TABLES))
        up, deleted = deltas.churn(m, np.random.default_rng(13))
        keep, uobj = deltas.objects_struct(up)
        e.apply_objects(uobj, deleted)
        e.diff()
        names = {s[0] for s in e.stage_timings()}
        assert not (actual_side & names)
        assert "classify_objects" in names


def _cuda_kernels(fn):
    """CUDA kernels that fn() launches, counted by torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in ev.name.lower()
               and "memset" not in ev.name.lower())


@pytest.mark.gpu
def test_gpu_apply_launches_fewer_kernels_than_reload(garecon):
    import importlib
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    deltas = importlib.import_module("aws-global-accelerator-controller_b200.deltas")
    snap = synth.generate(3, 20_000)
    with garecon.Engine(cluster_name=snap.cluster) as e:
        e.load(snap)
        e.diff()
        m = deltas.ColumnMirror(garecon.tables.columns(snap.objects, garecon.tables.OBJ_TABLES))
        up, deleted = deltas.churn(m, np.random.default_rng(14))
        keep, uobj = deltas.objects_struct(up)
        rows, _, _ = m.apply(up, deleted)
        msnap = m.snapshot(garecon.tables.columns(snap.actual, garecon.tables.ACT_TABLES))
        res = {}

        def apply_then_keys():
            e.apply_objects(uobj, deleted)
            res["apply"] = e.diff_keys(rows.tolist(), deleted)

        def load_then_keys():
            e.load(msnap)
            res["load"] = e.diff_keys(rows.tolist(), deleted)

        n_apply = _cuda_kernels(apply_then_keys)
        n_load = _cuda_kernels(load_then_keys)
    assert res["apply"].diff(res["load"]) == []
    assert 0 < n_apply < n_load, (n_apply, n_load)
