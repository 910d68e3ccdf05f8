"""gar_snapshot_export: the resident tables exported to host memory in the compacted layout.

Every exported column and slab is compared with the numpy statement of the compaction (deltas.compact / deltas.compact_actual of
the tables the engine holds), and the export is loaded into a second engine whose answers must equal the source engine's and
the oracle's.  The cases run on the host simulation (CPU tier) and on the GPU."""
import ctypes as C
import importlib
import random

import numpy as np
import pytest

import egbcases
import randmodel
from test_actual_deltas import AwsEvents, check_all
from test_object_deltas import Events, assert_same_full
from test_slab_compaction import skewed_model, with_columns
from test_zone_deltas import State, ZoneEvents

OBJ, ACT, BOTH = 1, 2, 3
shard = importlib.import_module("aws-global-accelerator-controller_b200.shard")


def mods(garecon):
    return importlib.import_module("aws-global-accelerator-controller_b200.deltas"), garecon.tables


def addr(p):
    return C.cast(p, C.c_void_p).value or 0


def expected(garecon, snap):
    """(object columns, AWS columns) a compaction of the tables of `snap` leaves: what an export must give."""
    deltas, tables = mods(garecon)
    return (deltas.compact(tables.columns(snap.objects, tables.OBJ_TABLES)), deltas.compact_actual(tables.columns(snap.actual, tables.ACT_TABLES)))


def check_layout(garecon, struct, tabs, base, nbytes):
    """Columns in struct order, each at the next 16-byte aligned offset from `base`, the slab last, ending at nbytes."""
    at = 0
    for t, (nf, cl) in tabs.items():
        n = getattr(struct, nf)
        for name, kind in cl:
            width = 4 if isinstance(kind, tuple) else {"u8": 1, "i32": 4, "str": 8}[kind]
            rows = n + 1 if isinstance(kind, tuple) else n
            assert addr(getattr(struct, name)) - base == at, name
            at = (at + rows * width + 15) & ~15
    assert addr(struct.slab) - base == at
    assert at + struct.slab_len == nbytes


def check_export(garecon, engine, snap, groups=BOTH, buf=None):
    """Export `groups`; the engine's resident tables equal those of `snap` row for row.  -> the export."""
    _, tables = mods(garecon)
    size = engine.export_size(groups)
    x = engine.export(groups, buf)
    want_o, want_a = expected(garecon, snap)
    base = x.buf.ctypes.data
    for bit, struct, want, tabs, nbytes, slab_len, at in ((OBJ, x.objects, want_o, tables.OBJ_TABLES, x.result.obj_bytes, x.result.obj_slab_len, 0),
                                                         (ACT, x.actual, want_a, tables.ACT_TABLES, x.result.act_bytes, x.result.act_slab_len, x.act_at)):
        if groups & bit:
            got = tables.columns(struct, tabs)
            assert set(got) == set(want)
            for k in want:
                assert np.array_equal(got[k], want[k]), k
            assert slab_len == struct.slab_len == len(want["slab"])
            check_layout(garecon, struct, tabs, base + at, nbytes)
        else:
            assert bytes(struct) == bytes(type(struct)()) and nbytes == slab_len == 0  # a group not selected: untouched
    assert (size.obj_bytes, size.act_bytes, size.obj_slab_len, size.act_slab_len) == (x.result.obj_bytes, x.result.act_bytes, x.result.obj_slab_len,
                                                                                      x.result.act_slab_len)
    return x


def resident(engine, obj_len, act_len):
    """The resident slabs, read back."""
    return engine.read_slab(OBJ, 0, obj_len), engine.read_slab(ACT, 0, act_len)


def diffs(engine, rows, deleted, bindings=None):
    full = engine.diff()
    dev = engine.diff_device()
    dev = (int(dev.n_objects), int(dev.n_ops), int(dev.n_lbi), int(dev.n_dports), list(dev.section_begin))
    keys = engine.diff_keys(rows, deleted)
    b = engine.bindings_diff(bindings).ops.tolist() if bindings is not None else None
    return full, dev, keys, b


def same_diffs(a, b):
    assert a[0].diff(b[0]) == [], a[0].describe_first_mismatch(b[0])
    assert a[1] == b[1]
    assert a[2].diff(b[2]) == [], a[2].describe_first_mismatch(b[2])
    assert a[3] == b[3]


# ------------------------------------------------------------------ the cases (engine = host simulation or GPU)

def case_layout(garecon, engine, seed, layout):
    objects, actual = randmodel.make(seed, n_objects=40)
    snap = garecon.pack(objects, actual, layout=layout, seed=seed)
    engine.load(snap)
    for groups in (OBJ, ACT, BOTH):
        check_export(garecon, engine, snap, groups)


def case_lifecycle(garecon, oracle, engine, seed, n_objects, n_batches, oracle_mode):
    """Object, AWS and zone deltas and compactions in random order; after every step the export equals the compaction of the
    mirrors, and a second engine loaded from it answers as the oracle does on the mirrors."""
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=n_objects, n_bindings=3 * n_objects)
    b = garecon.pack_bindings(bindings, known)
    s = State(garecon, oracle, engine, objects, actual, oracle_mode)
    oev, aev, zev = Events(seed, actual), AwsEvents(seed), ZoneEvents(seed)
    rng = random.Random(seed * 13 + 1)
    restored = type(engine)(cluster_name="default", lib=engine.lib)
    try:
        for step in range(n_batches):
            c = rng.random()
            if c < 0.35:
                upserts, deleted = oev.batch(s.om.objects)
                usnap = garecon.pack(upserts, None) if upserts else None
                engine.apply_objects(usnap.objects if usnap else None, deleted)
                s.om.apply(upserts, deleted, usnap)
            elif c < 0.6:
                s.aws(aev.batch(s.model.actual))
            elif c < 0.8:
                s.zones(*zev.batch(s.model.actual["zones"]))
            else:
                groups = rng.choice([OBJ, ACT, BOTH])
                res = engine.compact(groups)
                if groups & OBJ:
                    s.om.slab = bytearray(engine.read_slab(OBJ, 0, res.obj_slab_len).tobytes())
                if groups & ACT:
                    s.model.slab_len = int(res.act_slab_len)
                    s.am.compact()
            msnap = s.msnap()
            x = check_export(garecon, engine, msnap, rng.choice([OBJ, ACT, BOTH]) if step % 3 else BOTH)
            if x.result.obj_bytes and x.result.act_bytes:
                restored.load(x)
                rows = rng.sample(range(len(s.om.objects)), min(len(s.om.objects), 6))
                xslab = np.ctypeslib.as_array(x.objects.slab, shape=(max(1, x.objects.slab_len),))[:x.objects.slab_len]
                assert_same_full(restored.diff(), oracle.diff(msnap, "default", mode=1), xslab, msnap.arrays["o.slab"])
                got, want = restored.diff_keys(rows, []), engine.diff_keys(rows, [])
                assert got.diff(want) == [], got.describe_first_mismatch(want)
        check_all(garecon, oracle, engine, s.om, s.model, b, list(range(0, len(s.om.objects), 3)), [], oracle_mode)
    finally:
        restored.close()


def case_changes_nothing(garecon, oracle, engine, seed):
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=30, n_bindings=90)
    snap = garecon.pack(objects, actual)
    b = garecon.pack_bindings(bindings, known)
    engine.load(snap)
    usnap = garecon.pack(objects[:5], None)
    grown = engine.apply_objects(usnap.objects, []).slab_len  # a grown object slab: the export differs from the resident bytes
    rows = list(range(0, len(objects), 4))
    deleted = [(0, "default/absent-export-0")]
    if seed % 2 == 0:
        diffs(engine, rows, deleted, b)  # prepared before the export for some seeds
    before_slabs = resident(engine, grown, snap.actual.slab_len)
    before = diffs(engine, rows, deleted, b)
    for groups in (OBJ, ACT, BOTH):
        engine.export(groups)
        after_slabs = resident(engine, grown, snap.actual.slab_len)
        assert all(np.array_equal(p, q) for p, q in zip(before_slabs, after_slabs))
        same_diffs(diffs(engine, rows, deleted, b), before)


def case_restore(garecon, oracle, engine, make_engine, seed, oracle_mode):
    """Export, load into a second engine, then the same deltas on both."""
    deltas, tables = mods(garecon)
    objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=40, n_bindings=120)
    b = garecon.pack_bindings(bindings, known)
    s = State(garecon, oracle, engine, objects, actual, oracle_mode)
    oev, aev, zev = Events(seed, actual), AwsEvents(seed), ZoneEvents(seed)
    for _ in range(3):  # grow both slabs
        upserts, deleted = oev.batch(s.om.objects)
        usnap = garecon.pack(upserts, None) if upserts else None
        engine.apply_objects(usnap.objects if usnap else None, deleted)
        s.om.apply(upserts, deleted, usnap)
        s.aws(aev.batch(s.model.actual))
    x = check_export(garecon, engine, s.msnap())
    e2 = make_engine()
    try:
        e2.load(x)
        msnap = s.msnap()
        rows = list(range(0, len(s.om.objects), 3))
        xslab = np.array(np.ctypeslib.as_array(x.objects.slab, shape=(max(1, x.objects.slab_len),))[:x.objects.slab_len])
        want = oracle.diff(msnap, "default", mode=1)
        assert_same_full(e2.diff(), want, xslab, msnap.arrays["o.slab"])
        assert_same_full(engine.diff(), want, s.om.slab, msnap.arrays["o.slab"])
        a2, a1 = diffs(e2, rows, [], b), diffs(engine, rows, [], b)
        assert a2[1] == a1[1] and a2[2].diff(a1[2]) == [] and a2[3] == a1[3]
        want_k = oracle.diff_keys(msnap, rows, [], mode=oracle_mode)
        assert a2[2].diff(want_k) == [], a2[2].describe_first_mismatch(want_k)
        # the same deltas on both: equal row results and answers; slab_base / slab_len once both slabs are compact
        for rnd in range(2):
            if rnd == 1:
                res = engine.compact(BOTH)
                e2.compact(BOTH)
                s.om.slab = bytearray(engine.read_slab(OBJ, 0, res.obj_slab_len).tobytes())
                s.model.slab_len = int(res.act_slab_len)
                s.am.compact()
            upserts, deleted = oev.batch(s.om.objects)
            usnap = garecon.pack(upserts, None) if upserts else None
            r1 = engine.apply_objects(usnap.objects if usnap else None, deleted)
            r2 = e2.apply_objects(usnap.objects if usnap else None, deleted)
            assert (r1.upsert_row.tolist(), r1.deleted_row.tolist(), r1.moved_from.tolist(), r1.n_objects) == (r2.upsert_row.tolist(), r2.deleted_row.tolist(),
                                                                                                             r2.moved_from.tolist(), r2.n_objects)
            assert rnd == 0 or (r1.slab_base, r1.slab_len) == (r2.slab_base, r2.slab_len)
            s.om.apply(upserts, deleted, usnap)
            e2_obj_len = r2.slab_len
            d = aev.batch(s.model.actual)
            r1 = s.aws(d)
            r2 = e2.apply_actual(d["_rows"].actual if d["_rows"] is not None else None, [t for t, _ in d.get("lbs", [])], [t for t, _ in d.get("accs", [])],
                                 [z for z, _ in d.get("zones", [])], d.get("lb_deleted", []), d.get("acc_deleted", []))
            assert tuple(r1)[:9] == tuple(r2)[:9] and (rnd == 0 or tuple(r1) == tuple(r2))
            added, zdel = zev.batch(s.model.actual["zones"])
            packed = garecon.pack([], {"zones": [z for _, z in added]}) if added else None
            r2 = e2.apply_zones(packed.actual if packed else None, [a for a, _ in added], zdel)
            r1, _ = s.zones(added, zdel)
            assert tuple(r1)[:3] == tuple(r2)[:3] and (rnd == 0 or tuple(r1) == tuple(r2))
            msnap = s.msnap()
            want = oracle.diff(msnap, "default", mode=1)
            assert_same_full(engine.diff(), want, s.om.slab, msnap.arrays["o.slab"])
            assert_same_full(e2.diff(), want, e2.read_slab(OBJ, 0, e2_obj_len), msnap.arrays["o.slab"])
            k1, k2 = engine.diff_keys(rows[:5], []), e2.diff_keys(rows[:5], [])
            assert k1.diff(k2) == [], k1.describe_first_mismatch(k2)
        # one exported group with a freshly packed table of the other
        fresh = garecon.pack(s.om.objects, s.model.actual)
        xa = check_export(garecon, engine, fresh, ACT)
        e2.load(type(x)(fresh.objects, xa.actual, xa.result, xa.buf, xa.act_at))
        assert_same_full(e2.diff(), oracle.diff(fresh, "default", mode=1), fresh.arrays["o.slab"], fresh.arrays["o.slab"])
        xo = check_export(garecon, engine, fresh, OBJ)
        e2.load(type(x)(xo.objects, fresh.actual, xo.result, xo.buf, 0))
        oslab = np.array(np.ctypeslib.as_array(xo.objects.slab, shape=(max(1, xo.objects.slab_len),))[:xo.objects.slab_len])
        assert_same_full(e2.diff(), oracle.diff(fresh, "default", mode=1), oslab, fresh.arrays["o.slab"])
    finally:
        e2.close()


def case_idempotent(garecon, engine, seed):
    objects, actual = randmodel.make(seed, n_objects=30)
    snap = garecon.pack(objects, actual, layout="shuffle", seed=seed)
    engine.load(snap)
    x1 = check_export(garecon, engine, snap)
    res = engine.compact(BOTH)
    x2 = check_export(garecon, engine, snap)
    assert x1.buf.tobytes() == x2.buf.tobytes()
    assert (res.obj_slab_len, res.act_slab_len) == (x2.result.obj_slab_len, x2.result.act_slab_len)
    assert engine.read_slab(OBJ, 0, res.obj_slab_len).tobytes() == bytes(C.string_at(x2.objects.slab, x2.objects.slab_len))
    assert engine.read_slab(ACT, 0, res.act_slab_len).tobytes() == bytes(C.string_at(x2.actual.slab, x2.actual.slab_len))


def case_sizes(garecon, engine):
    abi = garecon.abi
    objects, actual = randmodel.make(61, n_objects=25)
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    need = engine.export_size(BOTH)
    x = check_export(garecon, engine, snap)
    assert (x.result.obj_bytes, x.result.act_bytes) == (need.obj_bytes, need.act_bytes)
    guard = 64
    for short_obj in (True, False):
        ob = np.full(int(need.obj_bytes) + guard, 0xAB, dtype=np.uint8)
        ab = np.full(int(need.act_bytes) + guard, 0xAB, dtype=np.uint8)
        ocap, acap = int(need.obj_bytes) - short_obj, int(need.act_bytes) - (not short_obj)
        o, a, res = abi.GarObjects(), abi.GarActual(), abi.GarExportResult()
        rc = engine.lib.gar_snapshot_export(engine._h, BOTH, C.c_void_p(ob.ctypes.data), ocap, C.byref(o), C.c_void_p(ab.ctypes.data), acap, C.byref(a), C.byref(res))
        assert rc == abi.GAR_E_INVALID
        assert (res.obj_bytes, res.act_bytes) == (need.obj_bytes, need.act_bytes)
        assert (ob[ocap:] == 0xAB).all() and (ab[acap:] == 0xAB).all()
    # a buffer of exactly the needed size, and a size query of one group next to an export of the other
    ob = np.zeros(int(need.obj_bytes), dtype=np.uint8)
    o, a, res = abi.GarObjects(), abi.GarActual(), abi.GarExportResult()
    rc = engine.lib.gar_snapshot_export(engine._h, BOTH, C.c_void_p(ob.ctypes.data), len(ob), C.byref(o), None, 0, C.byref(a), C.byref(res))
    assert rc == 0 and bytes(a) == bytes(abi.GarActual()) and res.act_bytes == need.act_bytes
    want_o, _ = expected(garecon, snap)
    assert np.array_equal(garecon.tables.columns(o, garecon.tables.OBJ_TABLES)["slab"], want_o["slab"])


def case_edges(garecon, oracle, make_engine):
    _, tables = mods(garecon)
    objects, actual = randmodel.make(21, n_objects=24)
    empty_ok = make_engine(allow_empty_cache=True)
    engine = make_engine()
    try:
        for snap in (garecon.pack([], actual), garecon.pack([], None)):  # no objects; no objects and no zones
            empty_ok.load(snap)
            x = check_export(garecon, empty_ok, snap)
            assert x.result.obj_slab_len == 0
        snap = garecon.pack(objects, None)
        engine.load(snap)
        check_export(garecon, engine, snap)

        def stray(o, a):  # flag-gated references: obj_ingress_class far outside the slab (a load does not check it), rec_alias_dns never live
            o["obj_ingress_class"][np.flatnonzero((o["obj_flags"] & 2) == 0)] = np.uint64((200 << 40) | (len(o["slab"]) + (1 << 30)))
            plain = np.flatnonzero(a["rec_has_alias"] == 0)
            if len(plain) and len(a["rec_name"]):
                a["rec_alias_dns"][plain] = a["rec_name"][0]
        snap = with_columns(garecon, garecon.pack(objects, actual), stray)
        engine.load(snap)
        check_export(garecon, engine, snap)

        def intern(o, a):  # interned strings: the export is larger than the resident slab
            o["ann_val"][:] = o["ann_val"][np.argmax(o["ann_val"] >> np.uint64(40))]
            a["tag_val"][:] = a["tag_val"][np.argmax(a["tag_val"] >> np.uint64(40))]
        snap = with_columns(garecon, garecon.pack(objects, actual), intern)
        engine.load(snap)
        x = check_export(garecon, engine, snap)
        assert x.result.obj_slab_len > snap.objects.slab_len and x.result.act_slab_len > snap.actual.slab_len
        e2 = make_engine()
        try:
            e2.load(x)
            oslab = np.array(np.ctypeslib.as_array(x.objects.slab, shape=(x.objects.slab_len,)))
            assert_same_full(e2.diff(), oracle.diff(snap, "default", mode=1), oslab, snap.arrays["o.slab"])
        finally:
            e2.close()
    finally:
        empty_ok.close()
        engine.close()


def case_long_strings(garecon, oracle, engine):
    """Strings longer than COMPACT_LONG, one of them 9 MiB: it spans several 4 MiB gather chunks and wraps no slot early."""
    objects, actual = skewed_model()
    objects[9].setdefault("annotations", {})["example.com/huge"] = "z" * (9 << 20) + "!"
    for layout in ("row", "shuffle"):
        snap = garecon.pack(objects, actual, layout=layout, seed=3)
        engine.load(snap)
        x = check_export(garecon, engine, snap)
        engine.load(x)
        oslab = np.array(np.ctypeslib.as_array(x.objects.slab, shape=(x.objects.slab_len,)))
        assert_same_full(engine.diff(), oracle.diff(snap, "default", mode=1), oslab, snap.arrays["o.slab"])


def case_errors(garecon, engine, make_engine, lib, device):
    abi = garecon.abi
    objects, actual = randmodel.make(41, n_objects=20)
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    before = engine.diff()

    def rc_of(groups, o=True, a=True):
        res = abi.GarExportResult()
        return engine.lib.gar_snapshot_export(engine._h, groups, None, 0, C.byref(abi.GarObjects()) if o else None, None, 0,
                                              C.byref(abi.GarActual()) if a else None, C.byref(res))
    assert [rc_of(g) for g in (0, 4, BOTH | 8)] == [abi.GAR_E_INVALID] * 3
    assert rc_of(OBJ, o=False) == rc_of(ACT, a=False) == rc_of(BOTH, a=False) == abi.GAR_E_INVALID
    assert rc_of(OBJ, a=False) == rc_of(ACT, o=False) == abi.GAR_OK  # the struct of a group not selected may be NULL
    assert engine.diff().diff(before) == []
    e = make_engine()
    try:
        with pytest.raises(garecon.GarError) as ei:
            e.export(BOTH)
        assert ei.value.rc == abi.GAR_E_STATE
        e.load(snap)
        e.shard_route(abi.GarShard(0, 1, 0, 0, 0, 0, 0, 0, 0), 1)
        with pytest.raises(garecon.GarError) as ei:
            e.export(OBJ)
        assert ei.value.rc == abi.GAR_E_STATE
    finally:
        e.close()
    # sharded sub-snapshots, eight shards, both exchanges
    for peers in (False, True):
        slices = shard.slice_model(objects, actual, 8)
        engines, keep = [], []
        try:
            for o, a, _ in slices:
                x = garecon.Engine(cluster_name="default", lib=lib)
                s = garecon.pack(o, a)
                x.load(s)
                engines.append(x)
                keep.append(s)
            if peers:
                shard.exchange_local_peers(engines, [s[2] for s in slices])
            else:
                shard.exchange_local(engines, [s[2] for s in slices], keep, device=device)
            for x in engines:
                with pytest.raises(garecon.GarError) as ei:
                    x.export(BOTH)
                assert ei.value.rc == abi.GAR_E_STATE
        finally:
            for x in engines:
                x.close()


# ------------------------------------------------------------------ CPU tier (host simulation)

@pytest.fixture(scope="module")
def hostlib(garecon):
    import __graft_entry__ as ge
    return garecon.abi.load_library(ge.build_hostsim())


@pytest.fixture(scope="module")
def hostsim(garecon, hostlib):
    e = garecon.Engine(cluster_name="default", lib=hostlib)
    yield e
    e.close()


def host_engine(garecon, lib):
    return lambda **kw: garecon.Engine(cluster_name="default", lib=lib, **kw)


@pytest.mark.parametrize("layout", ["row", "level", "reverse", "shuffle"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_hostsim_layout_byte_for_byte(garecon, hostsim, seed, layout):
    case_layout(garecon, hostsim, seed, layout)


@pytest.mark.parametrize("seed", range(8))
def test_hostsim_lifecycle(garecon, oracle, hostsim, seed):
    case_lifecycle(garecon, oracle, hostsim, seed, 30, 10, 0)


@pytest.mark.parametrize("seed", range(3))
def test_hostsim_export_changes_nothing(garecon, oracle, hostsim, seed):
    case_changes_nothing(garecon, oracle, hostsim, seed)


@pytest.mark.parametrize("seed", range(3))
def test_hostsim_restore(garecon, oracle, hostsim, hostlib, seed):
    case_restore(garecon, oracle, hostsim, host_engine(garecon, hostlib), seed, 0)


def test_hostsim_idempotent(garecon, hostsim):
    case_idempotent(garecon, hostsim, 71)


def test_hostsim_sizes_and_buffers(garecon, hostsim):
    case_sizes(garecon, hostsim)


def test_hostsim_edges(garecon, oracle, hostlib):
    case_edges(garecon, oracle, host_engine(garecon, hostlib))


def test_hostsim_long_strings(garecon, oracle, hostsim):
    case_long_strings(garecon, oracle, hostsim)


def test_hostsim_state_and_errors(garecon, hostsim, hostlib):
    case_errors(garecon, hostsim, host_engine(garecon, hostlib), hostlib, "cpu")


def test_ctypes_export_struct_size_matches_header(garecon):
    import subprocess
    import tempfile
    from pathlib import Path
    repo = Path(__file__).resolve().parent.parent
    src = '#include <stdio.h>\n#include "garecon.h"\nint main(void) { printf("%zu\\n", sizeof(gar_export_result)); return 0; }\n'
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "s.c").write_text(src)
        subprocess.run(["gcc", "-I", str(repo / "include"), "-o", f"{d}/s", f"{d}/s.c"], check=True)
        out = subprocess.run([f"{d}/s"], capture_output=True, text=True, check=True).stdout.split()
    assert int(out[0]) == C.sizeof(garecon.abi.GarExportResult)


# ------------------------------------------------------------------ GPU tier

def gpu_engine(garecon):
    return lambda **kw: garecon.Engine(cluster_name="default", **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["row", "level", "reverse", "shuffle"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_gpu_layout_byte_for_byte(garecon, engine, seed, layout):
    case_layout(garecon, engine, seed, layout)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(700, 706))
def test_gpu_lifecycle(garecon, oracle, engine, seed):
    case_lifecycle(garecon, oracle, engine, seed, 60, 10, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_gpu_export_changes_nothing(garecon, oracle, engine, seed):
    case_changes_nothing(garecon, oracle, engine, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_gpu_restore(garecon, oracle, engine, seed):
    case_restore(garecon, oracle, engine, gpu_engine(garecon), seed, 1)


@pytest.mark.gpu
def test_gpu_idempotent(garecon, engine):
    case_idempotent(garecon, engine, 71)


@pytest.mark.gpu
def test_gpu_sizes_and_buffers(garecon, engine):
    case_sizes(garecon, engine)


@pytest.mark.gpu
def test_gpu_edges(garecon, oracle):
    case_edges(garecon, oracle, gpu_engine(garecon))


@pytest.mark.gpu
def test_gpu_long_strings(garecon, oracle, engine):
    case_long_strings(garecon, oracle, engine)


@pytest.mark.gpu
def test_gpu_state_and_errors(garecon, engine):
    case_errors(garecon, engine, gpu_engine(garecon), garecon.abi.load_library(), "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("no_graph", [False, True])
def test_gpu_launch_replay_survives_export(garecon, monkeypatch, no_graph):
    """Diff until replayed, export: the next diff still replays, and gar_diff_keys issues as many launches as before."""
    if no_graph:
        monkeypatch.setenv("GAR_NO_GRAPH", "1")
    objects, actual = randmodel.make(51, n_objects=60)
    snap = garecon.pack(objects, actual)
    with garecon.Engine(cluster_name="default") as e:
        e.load(snap)
        e.diff()
        k0 = e.diff_keys([1, 5, 9])  # on the prepared snapshot; a partial diff makes the next full diff record anew
        for _ in range(4):
            want = e.diff()
        assert e.counters()["launch_mode"] == (0 if no_graph else 2)
        for groups in (OBJ, ACT, BOTH):
            check_export(garecon, e, snap, groups)
            got = e.diff()
            assert got.diff(want) == []
            assert e.counters()["launch_mode"] == (0 if no_graph else 2)
        k = e.diff_keys([1, 5, 9])
        assert k.diff(k0) == [] and k.kernel_launches == k0.kernel_launches


@pytest.mark.gpu
def test_gpu_pinned_and_pageable_give_the_same_bytes(garecon, engine):
    import torch
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, 100_000)
    engine.load(snap)
    need = engine.export_size(BOTH)
    n = ((int(need.obj_bytes) + 15) & ~15) + int(need.act_bytes)
    pinned = torch.empty(n, dtype=torch.uint8, pin_memory=True).numpy()
    pinned[:] = 0  # the alignment gaps between columns are not written: start both buffers equal there
    a = engine.export(BOTH, pinned)
    b = check_export(garecon, engine, snap)
    assert a.buf.tobytes() == b.buf.tobytes()


@pytest.mark.gpu
def test_gpu_attached_snapshot(garecon, oracle):
    """An attached snapshot can be exported (the call only reads), with its slabs 16-byte aligned and 8 bytes past a boundary."""
    import torch
    tables = garecon.tables
    objects, actual = randmodel.make(5, n_objects=40)
    snap = garecon.pack(objects, actual, layout="shuffle", seed=5)
    for shift in (0, 8):
        keep = []

        def dev(struct, tabs):
            s = type(struct)()
            C.pointer(s)[0] = struct
            for t, (nf, cl) in tabs.items():
                for name, kind in cl:
                    arr = tables.columns(struct, {t: (nf, [(name, kind)])})[name]
                    x = torch.from_numpy(np.ascontiguousarray(arr).copy() if arr.size else np.zeros(1, dtype=arr.dtype)).cuda()
                    keep.append(x)
                    setattr(s, name, C.cast(C.c_void_p(x.data_ptr()), type(getattr(s, name))))
            sl = torch.zeros(shift + struct.slab_len + 64, dtype=torch.uint8, device="cuda")
            sl[shift:shift + struct.slab_len] = torch.from_numpy(np.array(tables.columns(struct, {})["slab"])).cuda()
            keep.append(sl)
            s.slab = C.cast(C.c_void_p(sl.data_ptr() + shift), type(s.slab))
            return s

        with garecon.Engine(cluster_name="default") as e:
            e.attach_device(dev(snap.objects, tables.OBJ_TABLES), dev(snap.actual, tables.ACT_TABLES))
            before = e.diff()
            x = check_export(garecon, e, snap)
            assert e.diff().diff(before) == []
            with garecon.Engine(cluster_name="default") as e2:
                e2.load(x)
                oslab = np.array(np.ctypeslib.as_array(x.objects.slab, shape=(x.objects.slab_len,)))
                assert_same_full(e2.diff(), oracle.diff(snap, "default", mode=1), oslab, snap.arrays["o.slab"])


@pytest.mark.gpu
def test_gpu_hot_txt_sets(garecon, oracle):
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(5, 200_000)
    with garecon.Engine(cluster_name=snap.cluster) as e:
        e.load(snap)
        x = check_export(garecon, e, snap)
        with garecon.Engine(cluster_name=snap.cluster) as e2:
            e2.load(x)
            got, want = e2.diff(), e.diff()
            oslab = np.array(np.ctypeslib.as_array(x.objects.slab, shape=(x.objects.slab_len,)))
            assert_same_full(got, want, oslab, garecon.tables.columns(snap.objects, garecon.tables.OBJ_TABLES)["slab"])


def pinned_buffer(engine, groups):
    import torch
    need = engine.export_size(groups)
    n = ((int(need.obj_bytes) + 15) & ~15) + int(need.act_bytes)
    buf = torch.empty(max(1, n), dtype=torch.uint8, pin_memory=True).numpy()
    buf[:] = 0
    return buf


@pytest.mark.gpu
@pytest.mark.parametrize("n_objects", [300_000, 1_000_000])
def test_gpu_large_object_group_next_to_tiny_aws_group_pinned(garecon, n_objects):
    """Both groups into pinned memory: the object group's last chunks are still on their way to the host when the AWS group's
    first chunks are gathered into the same ring slots.  Every byte must equal the mirrors' compaction, over repeated exports."""
    _, tables = mods(garecon)
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    big = synth.generate(3, n_objects)
    tiny = garecon.pack([], randmodel.make(5, n_objects=4)[1])
    snap = tables.from_columns(tables.columns(big.objects, tables.OBJ_TABLES), tables.columns(tiny.actual, tables.ACT_TABLES))
    with garecon.Engine(cluster_name=big.cluster) as e:
        e.load(snap)
        buf = pinned_buffer(e, BOTH)
        for _ in range(3):
            x = check_export(garecon, e, snap, BOTH, buf)
            assert x.result.obj_slab_len > 8 * 128 * 32 * 1024 and x.result.act_slab_len < 64 * 1024  # many object chunks, one AWS chunk


@pytest.mark.gpu
@pytest.mark.parametrize("n_objects", [100_000, 1_000_000])
def test_gpu_churn_then_export_at_scale(garecon, oracle, engine, n_objects):
    """configs[2] after churn batches: the export spans many ring chunks and wraps the ring; it equals the mirrors' compaction,
    and an engine loaded from it answers as the oracle does on the mirrors."""
    deltas, tables = mods(garecon)
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, n_objects)
    engine.load(snap)
    om = deltas.ColumnMirror(tables.columns(snap.objects, tables.OBJ_TABLES))
    am = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    rng = np.random.default_rng(n_objects + 1)
    for b in range(3):
        up, deleted = deltas.churn(om, rng, serial=b)
        keep, uobj = deltas.objects_struct(up)
        engine.apply_objects(uobj, deleted)
        om.apply(up, deleted)
        d = deltas.aws_churn(am, rng)
        keep2, arows = deltas.actual_struct(d["rows"])
        engine.apply_actual(arows, d["lb_target"], d["acc_target"], d["zone_target"], d["lb_deleted"], d["acc_deleted"])
        am.apply(**d)
    x = engine.export(BOTH, pinned_buffer(engine, BOTH))  # pinned: the copy stream runs behind the gather
    om.compact()
    am.compact()
    assert x.result.act_slab_len > 4 * 4 * 32 * 1024 * 128 or n_objects < 1_000_000  # more than a full turn of the ring
    for struct, want, tabs in ((x.objects, om.cur, tables.OBJ_TABLES), (x.actual, am.cur, tables.ACT_TABLES)):
        got = tables.columns(struct, tabs)
        for k in want:
            assert np.array_equal(got[k], want[k]), k
    msnap = tables.from_columns(om.cur, am.cur)
    with garecon.Engine(cluster_name=snap.cluster) as e2:
        e2.load(x)
        got = e2.diff()
        want = oracle.diff(msnap, snap.cluster, mode=1, threads=8)
        assert got.diff(want) == [], got.describe_first_mismatch(want)  # the exported slab is the mirror's: tok refs match bit for bit
