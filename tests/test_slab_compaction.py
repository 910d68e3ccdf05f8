"""Slab compaction (gar_snapshot_compact) and gar_snapshot_read_slab.

The compacted slabs are compared byte for byte with the numpy statement of the layout (deltas.compact / deltas.compact_actual of
the resident tables), and every kind of diff after a compaction with the oracle: tok_name / tok_region as the strings they name
(read back through gar_snapshot_read_slab), everything else bit for bit.  The cases run on the host simulation (CPU tier) and on
the GPU."""
import copy
import importlib
import random
import time

import numpy as np
import pytest

import egbcases
import randmodel
from test_actual_deltas import AwsEvents, AwsModel, apply_delta
from test_object_deltas import Events, Mirror, assert_same_full, key_of

OBJ, ACT, BOTH = 1, 2, 3


def mods(garecon):
    return importlib.import_module("aws-global-accelerator-controller_b200.deltas"), garecon.tables


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


def live_slabs(garecon, snap):
    """(object slab, AWS slab) a compaction of both groups must leave for the tables of `snap`."""
    deltas, tables = mods(garecon)
    return (deltas.compact(tables.columns(snap.objects, tables.OBJ_TABLES))["slab"],
            deltas.compact_actual(tables.columns(snap.actual, tables.ACT_TABLES))["slab"])


def compact_and_check(garecon, engine, snap, groups=BOTH):
    """Compact `groups` of the engine, whose resident tables equal those of `snap` row for row; the selected slabs must be the
    live strings of `snap`, byte for byte.  -> (result, resident object slab bytes)."""
    res = engine.compact(groups)
    want_o, want_a = live_slabs(garecon, snap)
    if groups & OBJ:
        assert res.obj_slab_len == len(want_o)
        assert np.array_equal(engine.read_slab(OBJ, 0, res.obj_slab_len), want_o)
    else:
        assert res.obj_slab_len == res.obj_slab_before
    if groups & ACT:
        assert res.act_slab_len == len(want_a)
        assert np.array_equal(engine.read_slab(ACT, 0, res.act_slab_len), want_a)
    else:
        assert res.act_slab_len == res.act_slab_before
    return res, engine.read_slab(OBJ, 0, res.obj_slab_len)


def check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, bindings=None, rows=(), deleted=(), cluster="default"):
    """Full, incremental and binding diffs of the engine equal the oracle's on `snap`; oslab: the resident object slab."""
    got = engine.diff()
    assert_same_full(got, oracle.diff(snap, cluster, mode=1), oslab, snap.arrays["o.slab"])
    rows = list(rows)
    got = engine.diff_keys(rows, list(deleted))
    want = oracle.diff_keys(snap, rows, list(deleted), cluster=cluster, mode=oracle_mode)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    if bindings is not None:
        assert engine.bindings_diff(bindings).ops.tolist() == oracle.bindings_diff(snap, bindings).ops.tolist()


# ------------------------------------------------------------------ the cases (engine = host simulation or GPU)

def case_layout(garecon, oracle, engine, seed, layout, oracle_mode):
    objects, actual = randmodel.make(seed, n_objects=40)
    snap = garecon.pack(objects, actual, layout=layout, seed=seed)
    engine.load(snap)
    res, oslab = compact_and_check(garecon, engine, snap)
    assert (res.obj_slab_before, res.act_slab_before) == (int(snap.objects.slab_len), int(snap.actual.slab_len))
    aslab = engine.read_slab(ACT, 0, res.act_slab_len)
    check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, rows=range(0, len(objects), 3))
    again, oslab2 = compact_and_check(garecon, engine, snap)  # idempotent: neither bytes nor lengths change
    assert (again.obj_slab_before, again.obj_slab_len, again.act_slab_before, again.act_slab_len) == (res.obj_slab_len, res.obj_slab_len, res.act_slab_len, res.act_slab_len)
    assert np.array_equal(oslab, oslab2) and np.array_equal(aslab, engine.read_slab(ACT, 0, again.act_slab_len))


def case_results_unchanged(garecon, oracle, engine, seed, groups, oracle_mode):
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=30, n_bindings=90)
    snap = garecon.pack(objects, actual)
    b = garecon.pack_bindings(bindings, known)
    engine.load(snap)
    rows = list(range(0, len(objects), 4))
    deleted = [(0, "default/absent-compact-0"), (1, "prod/absent-compact-1")]
    if seed % 2 == 0:  # a prepared snapshot for some seeds (digests, indexes and owner indexes resident), a fresh one for the others
        check_diffs(garecon, oracle, engine, snap, snap.arrays["o.slab"], oracle_mode, b, rows, deleted)
    _, oslab = compact_and_check(garecon, engine, snap, groups)
    check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, b, rows, deleted)


def case_interleaving(garecon, oracle, engine, seed, n_objects, n_batches, oracle_mode):
    """Object and AWS deltas with a compaction of a random group mask after random batches: after every step the engine equals a
    fresh load of the mirror, and slab_base / slab_len of later deltas follow the compacted lengths."""
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=n_objects, n_bindings=3 * n_objects)
    snap = garecon.pack(objects, actual)
    b = garecon.pack_bindings(bindings, known)
    engine.load(snap)
    om, model = Mirror(objects, snap), AwsModel(actual, snap)
    oev, aev = Events(seed, actual), AwsEvents(seed)
    rng = random.Random(seed * 7 + 3)
    if seed % 3 == 0:
        engine.diff()
    compactions = 0
    for step in range(n_batches):
        if rng.random() < 0.6:
            upserts, deleted = oev.batch(om.objects)
            usnap = garecon.pack(upserts, None) if upserts else None
            res = engine.apply_objects(usnap.objects if usnap else None, deleted)
            up_row, del_row, moved, base = om.apply(upserts, deleted, usnap)
            assert (res.upsert_row.tolist(), res.deleted_row.tolist(), res.moved_from.tolist()) == (up_row, del_row, moved)
            assert res.slab_len == len(om.slab) and (not upserts or res.slab_base == base)
        if rng.random() < 0.6:
            apply_delta(garecon, engine, model, aev.batch(model.actual))  # checks slab_base / slab_len against model.slab_len
        msnap = garecon.pack(om.objects, model.actual)
        if rng.random() < 0.6 or step == n_batches - 2:
            groups = rng.choice([OBJ, ACT, BOTH])
            want_o, want_a = live_slabs(garecon, msnap)
            res, oslab = compact_and_check(garecon, engine, msnap, groups)
            assert (res.obj_slab_before, res.act_slab_before) == (len(om.slab), model.slab_len)
            if groups & OBJ:
                assert res.obj_slab_before >= res.obj_slab_len == len(want_o)
                om.slab = bytearray(oslab.tobytes())
            if groups & ACT:
                assert res.act_slab_before >= res.act_slab_len == len(want_a)
                model.slab_len = int(res.act_slab_len)
            compactions += 1
        rows = rng.sample(range(len(om.objects)), min(len(om.objects), 8))
        gone = [k for k in (key_of(o) for o in rng.sample(objects, 2)) if k not in {key_of(o) for o in om.objects}]
        check_diffs(garecon, oracle, engine, msnap, om.slab, oracle_mode, b, rows, gone)
    assert compactions


def case_dead_strings_are_dropped(garecon, engine):
    """Replacing every object and every accelerator leaves their old strings behind: slab_len before a compaction is strictly larger
    than the live size, after it equal."""
    objects, actual = randmodel.make(11, n_objects=25)
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    usnap = garecon.pack(objects, None)
    res = engine.apply_objects(usnap.objects, [])
    assert res.slab_len > int(snap.objects.slab_len)
    rows = garecon.pack([], {"accelerators": actual["accelerators"]})
    ares = engine.apply_actual(rows.actual, acc_target=list(range(len(actual["accelerators"]))))
    assert ares.slab_len > int(snap.actual.slab_len)
    c, _ = compact_and_check(garecon, engine, snap)
    assert (c.obj_slab_before, c.act_slab_before) == (res.slab_len, ares.slab_len)
    assert c.obj_slab_len < c.obj_slab_before and c.act_slab_len < c.act_slab_before
    res = engine.apply_objects(usnap.objects, [])  # the next delta appends behind the compacted slab
    assert res.slab_base == (c.obj_slab_len + 15) & ~15 and res.slab_len == res.slab_base + int(usnap.objects.slab_len)


def with_columns(garecon, snap, edit):
    """`snap` rebuilt from its columns after edit(o_cols, a_cols) changed them."""
    _, tables = mods(garecon)
    o = {k: np.array(v, copy=True) for k, v in tables.columns(snap.objects, tables.OBJ_TABLES).items()}
    a = {k: np.array(v, copy=True) for k, v in tables.columns(snap.actual, tables.ACT_TABLES).items()}
    edit(o, a)
    return tables.from_columns(o, a)


def case_edges(garecon, oracle, make_engine, oracle_mode):
    _, tables = mods(garecon)
    objects, actual = randmodel.make(21, n_objects=24)
    empty_ok = make_engine(allow_empty_cache=True)
    engine = make_engine()
    try:
        # no objects and a non-empty AWS side; objects and no AWS rows
        snap = garecon.pack([], actual)
        empty_ok.load(snap)
        _, oslab = compact_and_check(garecon, empty_ok, snap)
        assert len(oslab) == 0
        assert_same_full(empty_ok.diff(), oracle.diff(snap, "default", mode=1), oslab, snap.arrays["o.slab"])
        snap = garecon.pack(objects, None)
        engine.load(snap)
        res, oslab = compact_and_check(garecon, engine, snap)
        assert res.act_slab_len == 0
        check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, rows=[0, 5])

        # every AWS string empty
        def blank(o, a):
            for t, (_, cl) in tables.ACT_TABLES.items():
                for name, kind in cl:
                    if kind == "str":
                        a[name][:] = 0
        snap = with_columns(garecon, garecon.pack(objects, actual), blank)
        engine.load(snap)
        res, oslab = compact_and_check(garecon, engine, snap)
        assert res.act_slab_len == 0
        check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, rows=[1, 2])

        # obj_ingress_class of a row without GAR_OBJ_HAS_INGRESS_CLASS may hold anything, also a reference far outside the slab
        # (gar_snapshot_load does not check it); rec_alias_dns of a record without an alias is inside the slab but never live
        def stray(o, a):
            rows = np.flatnonzero((o["obj_flags"] & 2) == 0)
            assert len(rows)
            o["obj_ingress_class"][rows] = np.uint64((200 << 40) | (len(o["slab"]) + (1 << 30)))
            plain = np.flatnonzero(a["rec_has_alias"] == 0)
            if len(plain) and len(a["rec_name"]):
                a["rec_alias_dns"][plain] = a["rec_name"][0]
        base = garecon.pack(objects, actual)
        snap = with_columns(garecon, base, stray)
        engine.load(snap)
        res, oslab = compact_and_check(garecon, engine, snap)
        assert (res.obj_slab_len, res.act_slab_len) == (int(base.objects.slab_len), int(base.actual.slab_len))
        check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, rows=range(0, 24, 5))

        # duplicate object keys in a load: obj_canon still resolves to the lowest row
        dup = copy.deepcopy(objects[2])
        dup["lb_ingress"] = []
        dobjects = objects[:9] + [dup] + objects[9:] + [copy.deepcopy(objects[2])]
        snap = garecon.pack(dobjects, actual)
        engine.load(snap)
        engine.diff()
        _, oslab = compact_and_check(garecon, engine, snap)
        check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, rows=[2, 9, len(dobjects) - 1])

        # interned input: many references to one string.  The compacted slab is larger; the answers are the same
        def intern(o, a):
            o["ann_val"][:] = o["ann_val"][np.argmax(o["ann_val"] >> np.uint64(40))]
            a["tag_val"][:] = a["tag_val"][np.argmax(a["tag_val"] >> np.uint64(40))]
        snap = with_columns(garecon, garecon.pack(objects, actual), intern)
        engine.load(snap)
        res, oslab = compact_and_check(garecon, engine, snap)
        assert res.obj_slab_len > res.obj_slab_before and res.act_slab_len > res.act_slab_before
        check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, rows=range(0, 24, 7))
    finally:
        empty_ok.close()
        engine.close()


def skewed_model():
    objects, actual = randmodel.make(31, n_objects=30)
    objects = copy.deepcopy(objects)
    actual = copy.deepcopy(actual)
    objects[7].setdefault("annotations", {})["example.com/blob"] = "x" * (3 << 20)  # spans 96 windows
    objects[8].setdefault("annotations", {})["example.com/kib"] = "abcdefghijklmnopq" * 61  # 1037 bytes: just over the long-string threshold
    zone = next(z for z in actual["zones"])
    zone.setdefault("records", []).append({"name": "big." + zone["name"], "type": "TXT", "values": ['"' + "y" * (1 << 20) + '"', '"short"']})
    return objects, actual


def case_skew(garecon, oracle, engine, oracle_mode):
    objects, actual = skewed_model()
    for layout in ("row", "shuffle"):  # shuffled: the long strings start at every phase of a 16-byte line
        snap = garecon.pack(objects, actual, layout=layout, seed=5)
        engine.load(snap)
        _, oslab = compact_and_check(garecon, engine, snap)
        check_diffs(garecon, oracle, engine, snap, oslab, oracle_mode, rows=[7, 8, 9])


def case_errors(garecon, oracle, engine, make_engine, oracle_mode):
    abi = garecon.abi
    objects, actual = randmodel.make(41, n_objects=20)
    snap = garecon.pack(objects, actual)
    engine.load(snap)

    def refused(fn, rc):
        with pytest.raises(garecon.GarError) as ei:
            fn()
        assert ei.value.rc == rc
        check_diffs(garecon, oracle, engine, snap, snap.arrays["o.slab"], oracle_mode, rows=[0, 3])

    refused(lambda: engine.compact(0), abi.GAR_E_INVALID)
    refused(lambda: engine.compact(4), abi.GAR_E_INVALID)
    refused(lambda: engine.compact(BOTH | 8), abi.GAR_E_INVALID)
    refused(lambda: engine.read_slab(BOTH, 0, 1), abi.GAR_E_INVALID)
    refused(lambda: engine.read_slab(OBJ, int(snap.objects.slab_len), 1), abi.GAR_E_INVALID)
    refused(lambda: engine.read_slab(ACT, 1 << 50, 0), abi.GAR_E_INVALID)
    assert len(engine.read_slab(OBJ, int(snap.objects.slab_len), 0)) == 0
    assert engine.read_slab(ACT, 3, 11).tobytes() == snap.arrays["a.slab"][3:14].tobytes()
    e = make_engine()
    try:
        for fn in (lambda: e.compact(BOTH), lambda: e.read_slab(OBJ, 0, 0)):
            with pytest.raises(garecon.GarError) as ei:
                fn()
            assert ei.value.rc == abi.GAR_E_STATE
        e.load(snap)
        e.shard_route(abi.GarShard(0, 1, 0, 0, 0, 0, 0, 0, 0), 1)
        with pytest.raises(garecon.GarError) as ei:
            e.compact(OBJ)
        assert ei.value.rc == abi.GAR_E_STATE
    finally:
        e.close()


# ------------------------------------------------------------------ CPU tier (host simulation)

def host_engine(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    return lambda **kw: garecon.Engine(cluster_name="default", lib=lib, **kw)


@pytest.mark.parametrize("layout", ["row", "level", "reverse", "shuffle"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_hostsim_layout_byte_for_byte(garecon, oracle, hostsim, seed, layout):
    case_layout(garecon, oracle, hostsim, seed, layout, 0)


@pytest.mark.parametrize("groups", [OBJ, ACT, BOTH])
@pytest.mark.parametrize("seed", range(4))
def test_hostsim_results_unchanged(garecon, oracle, hostsim, seed, groups):
    case_results_unchanged(garecon, oracle, hostsim, seed, groups, 0)


@pytest.mark.parametrize("seed", range(12))
def test_hostsim_interleaving(garecon, oracle, hostsim, seed):
    case_interleaving(garecon, oracle, hostsim, seed, 30, random.Random(seed).randrange(5, 10), 0)


def test_hostsim_interleaving_with_tiny_capacities(garecon, oracle, hostsim, monkeypatch):
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    case_interleaving(garecon, oracle, hostsim, 77, 30, 6, 0)


def test_hostsim_dead_strings_are_dropped(garecon, hostsim):
    case_dead_strings_are_dropped(garecon, hostsim)


def test_hostsim_edge_rows(garecon, oracle):
    case_edges(garecon, oracle, host_engine(garecon), 0)


def test_hostsim_skew(garecon, oracle, hostsim):
    case_skew(garecon, oracle, hostsim, 0)


def test_hostsim_state_and_errors(garecon, oracle, hostsim):
    case_errors(garecon, oracle, hostsim, host_engine(garecon), 0)


def test_hostsim_table_churn_then_compact(garecon, oracle, hostsim):
    """deltas.churn / aws_churn batches, then a compaction: the engine's slabs are the mirrors' after their compact()."""
    churn_and_compact(garecon, oracle, hostsim, 3000, 1)


def churn_and_compact(garecon, oracle, engine, n_objects, threads):
    deltas, tables = mods(garecon)
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, n_objects)
    engine.load(snap)
    om = deltas.ColumnMirror(tables.columns(snap.objects, tables.OBJ_TABLES))
    am = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    rng = np.random.default_rng(n_objects)
    for b in range(3):
        up, deleted = deltas.churn(om, rng, serial=b)
        keep, uobj = deltas.objects_struct(up)
        engine.apply_objects(uobj, deleted)
        rows, _, _ = om.apply(up, deleted)
        d = deltas.aws_churn(am, rng)
        keep2, arows = deltas.actual_struct(d["rows"])
        engine.apply_actual(arows, d["lb_target"], d["acc_target"], d["zone_target"], d["lb_deleted"], d["acc_deleted"])
        am.apply(**d)
    grown = (om.slab_len, am.slab_len)
    res = engine.compact(BOTH)
    assert (res.obj_slab_before, res.act_slab_before) == grown
    assert (res.obj_slab_len, res.act_slab_len) == (om.compact(), am.compact())
    assert np.array_equal(engine.read_slab(OBJ, 0, res.obj_slab_len), om.cur["slab"])
    assert np.array_equal(engine.read_slab(ACT, 0, res.act_slab_len), am.cur["slab"])
    msnap = tables.from_columns(om.cur, am.cur)
    got = engine.diff()
    want = oracle.diff(msnap, snap.cluster, mode=1, threads=threads)
    assert got.diff(want) == [], got.describe_first_mismatch(want)  # the mirror's slab is the resident one: tok refs match bit for bit
    got = engine.diff_keys(rows.tolist(), deleted)
    want = oracle.diff_keys(msnap, rows.tolist(), deleted, cluster=snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    up, deleted = deltas.churn(om, rng, serial=9)  # a delta after the compaction lands behind the compacted slab
    keep, uobj = deltas.objects_struct(up)
    r = engine.apply_objects(uobj, deleted)
    om.apply(up, deleted)
    assert r.slab_base == (res.obj_slab_len + 15) & ~15 and r.slab_len == om.slab_len


def test_ctypes_compact_struct_size_matches_header(garecon):
    import ctypes
    import subprocess
    import tempfile
    from pathlib import Path
    repo = Path(__file__).resolve().parent.parent
    src = '#include <stdio.h>\n#include "garecon.h"\nint main(void) { printf("%zu %d %d\\n", sizeof(gar_compact_result), GAR_COMPACT_OBJECTS, GAR_COMPACT_ACTUAL); return 0; }\n'
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(repo / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout.split()
    assert [int(x) for x in out] == [ctypes.sizeof(garecon.abi.GarCompactResult), garecon.abi.COMPACT_OBJECTS, garecon.abi.COMPACT_ACTUAL]


# ------------------------------------------------------------------ GPU tier

def gpu_engine(garecon):
    return lambda **kw: garecon.Engine(cluster_name="default", **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["row", "level", "reverse", "shuffle"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_gpu_layout_byte_for_byte(garecon, oracle, engine, seed, layout):
    case_layout(garecon, oracle, engine, seed, layout, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("groups", [OBJ, ACT, BOTH])
@pytest.mark.parametrize("seed", range(4))
def test_gpu_results_unchanged(garecon, oracle, engine, seed, groups):
    case_results_unchanged(garecon, oracle, engine, seed, groups, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(600, 610))
def test_gpu_interleaving(garecon, oracle, engine, seed):
    case_interleaving(garecon, oracle, engine, seed, 80, random.Random(seed).randrange(5, 10), 1)


@pytest.mark.gpu
def test_gpu_dead_strings_are_dropped(garecon, engine):
    case_dead_strings_are_dropped(garecon, engine)


@pytest.mark.gpu
def test_gpu_edge_rows(garecon, oracle):
    case_edges(garecon, oracle, gpu_engine(garecon), 1)


@pytest.mark.gpu
def test_gpu_skew(garecon, oracle, engine):
    case_skew(garecon, oracle, engine, 1)


@pytest.mark.gpu
def test_gpu_state_and_errors(garecon, oracle, engine):
    case_errors(garecon, oracle, engine, gpu_engine(garecon), 1)


@pytest.mark.gpu
def test_gpu_attached_snapshot_is_a_state_error(garecon):
    import ctypes
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
            e.compact(BOTH)
        assert ei.value.rc == garecon.abi.GAR_E_STATE
        assert e.diff().diff(before) == []
        assert e.read_slab(OBJ, 0, 16).tobytes() == snap.arrays["o.slab"][:16].tobytes()  # reading an attached slab is allowed


@pytest.mark.gpu
@pytest.mark.parametrize("no_graph", [False, True])
def test_gpu_launch_replay_after_compaction(garecon, oracle, monkeypatch, no_graph):
    """Diff until replayed, compact: the next diff is eager and equal, later ones are recorded and replayed again."""
    if no_graph:
        monkeypatch.setenv("GAR_NO_GRAPH", "1")
    objects, actual = randmodel.make(51, n_objects=60)
    snap = garecon.pack(objects, actual)
    want = oracle.diff(snap, "default", mode=1)
    with garecon.Engine(cluster_name="default") as e:
        e.load(snap)
        oslab = snap.arrays["o.slab"]
        for groups in (OBJ, ACT, BOTH):
            modes = []
            for _ in range(4):
                assert_same_full(e.diff(), want, oslab, snap.arrays["o.slab"])
                modes.append(e.counters()["launch_mode"])
            assert modes[-1] == (0 if no_graph else 2), modes
            _, oslab = compact_and_check(garecon, e, snap, groups)
            assert_same_full(e.diff(), want, oslab, snap.arrays["o.slab"])
            assert e.counters()["launch_mode"] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("n_objects", [100_000, 1_000_000])
def test_gpu_churn_then_compact_at_scale(garecon, oracle, engine, n_objects):
    churn_and_compact(garecon, oracle, engine, n_objects, 8)


@pytest.mark.gpu
def test_gpu_hot_txt_sets_no_cliff(garecon, oracle):
    """Config 5 (TXT sets of 10^5 values) against config 2 at the same object count: correct, and the compaction of the skewed
    snapshot takes no more per byte than a small multiple of the unskewed one (not a benchmark: a bound that catches a thread or
    block walking a whole hot set)."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    per_byte = {}
    for cfg in (2, 5):
        snap = synth.generate(cfg, 200_000)
        with garecon.Engine(cluster_name=snap.cluster) as e:
            e.load(snap)
            e.compact(BOTH)  # first use: buffers are allocated
            best = 1e9
            for _ in range(3):
                t0 = time.perf_counter()
                res = e.compact(BOTH)  # returns after a device synchronise
                best = min(best, time.perf_counter() - t0)
            want_o, want_a = live_slabs(garecon, snap)
            assert np.array_equal(e.read_slab(OBJ, 0, res.obj_slab_len), want_o) and np.array_equal(e.read_slab(ACT, 0, res.act_slab_len), want_a)
            got = e.diff()
            ref = oracle.diff(snap, snap.cluster, mode=1, threads=8)
            assert_same_full(got, ref, want_o, garecon.tables.columns(snap.objects, garecon.tables.OBJ_TABLES)["slab"])
            per_byte[cfg] = best / (res.obj_slab_len + res.act_slab_len)
    assert per_byte[5] < 10 * per_byte[2], per_byte
