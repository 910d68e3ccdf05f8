"""GPU tier: the adversarial models of tests/scalemodels.py at 10^4-6*10^4 objects, every entry point against the oracle.

At the sizes of the other model tests (40-400 objects) a row pass is one or two blocks and every index build, scan and
compaction fits in one tile; the generator configs of test_gpu_large.py reach 10^5-10^6 objects but are regular.  Here the
decision kernels see bad hostnames, duplicate chains, orphans by the thousand and hot zones across many blocks, tiles and
warps: the full diff through its eager, recorded and replayed launches, the device-resident result byte for byte,
gar_diff_keys with deleted keys, gar_bindings_diff with thousands of endpoint groups, the GAR_NO_TMA / GAR_TMA_ALL /
GAR_TINY_CAPS engine forms, eight shards on one GPU, and snapshots attached from caller-owned device buffers (slabs 16-byte
aligned and 8 bytes past a 16-byte boundary)."""
import ctypes
import importlib
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest

import scalemodels
from test_backend_kernels import engine_in_form
from test_sharded import check_slices

pytestmark = pytest.mark.gpu

shard = importlib.import_module("aws-global-accelerator-controller_b200.shard")

THREADS = os.cpu_count() or 4
SLAB_PAD = 32  # readable bytes the engine needs behind an attached slab (include/garecon.h gar_snapshot_attach_device)


def _deleted_sample(objects, seed, frac=0.02):
    """Keys of a seeded sample of objects that are still in the cache, plus keys that match nothing."""
    rng = random.Random(seed)
    return [scalemodels.key_of(o) for o in rng.sample(objects, int(len(objects) * frac))] + scalemodels.ABSENT_KEYS


def _make(name):
    """-> (objects, actual, deleted keys, bindings or None, known endpoint groups or None)."""
    if name == "rand":
        objects, actual, dropped = scalemodels.randmodel_dropped(11, 60_000, frac=0.08)
        return objects, actual, dropped + scalemodels.ABSENT_KEYS, None, None
    if name == "multilbi":
        objects, actual = scalemodels.multilbi_cluster(3, 20_000)
        return objects, actual, _deleted_sample(objects, 3), None, None
    if name == "hot":
        objects, actual = scalemodels.hot_cluster(4, 10_000)
        deleted = _deleted_sample(objects, 4) + [(0, "default/hot"), (0, "default/left-the-cache"), (1, "default/unannotated")]
        return objects, actual, deleted, None, None
    if name == "bindings":
        objects, actual, bindings, known = scalemodels.bindings_cluster(5, 20_000, 100_000, n_known=4000)
        return objects, actual, _deleted_sample(objects, 5), bindings, known
    raise KeyError(name)


class Models:
    """Each model built, packed and diffed by the oracle once per module, on first use."""

    def __init__(self, garecon, oracle):
        self.garecon, self.oracle, self.cache = garecon, oracle, {}

    def __call__(self, name, layout="row"):
        if (name, layout) not in self.cache:
            if name not in self.cache:
                self.cache[name] = _make(name)
            objects, actual, deleted, bindings, known = self.cache[name]
            snap = self.garecon.pack(objects, actual, layout=layout)
            self.cache[name, layout] = SimpleNamespace(
                name=name, objects=objects, actual=actual, deleted=deleted, snap=snap, want=self.oracle.diff(snap, "default", mode=1, threads=THREADS),
                bindings=self.garecon.pack_bindings(bindings, known) if bindings is not None else None)
        return self.cache[name, layout]


@pytest.fixture(scope="module")
def models(garecon, oracle):
    return Models(garecon, oracle)


MODELS = ["rand", "multilbi", "hot", "bindings"]


def _batches(n, seed):
    """(id, rows) for batches of 1 %, 10 % and 100 % of the rows, each sorted and shuffled."""
    rng = random.Random(seed)
    out = []
    for pct in (1, 10, 100):
        rows = sorted(rng.sample(range(n), max(1, n * pct // 100)))
        out.append((f"{pct}%-sorted", rows))
        shuffled = list(rows)
        rng.shuffle(shuffled)
        out.append((f"{pct}%-shuffled", shuffled))
    return out


def check_against_full(inc, full, rows):
    """test_incremental._check_against_full for batches of any size: the object-section ops of the incremental result are the
    full diff's ops of those rows, rows in batch order and each row's ops in their full-diff order; the statuses follow rows."""
    rows = np.asarray(rows, dtype=np.int64)
    pos = np.full(int(full.n_objects), -1, dtype=np.int64)
    pos[rows] = np.arange(len(rows))
    sb, isb = [int(x) for x in full.section_begin], [int(x) for x in inc.section_begin]
    for sec in (0, 2):
        fops = full.ops[sb[sec]:sb[sec + 1]]
        p = pos[fops["obj"].astype(np.int64)]
        want = fops[p >= 0][np.argsort(p[p >= 0], kind="stable")]
        got = inc.ops[isb[sec]:isb[sec + 1]]
        assert np.array_equal(got, want), (sec, len(got), len(want))
    assert np.array_equal(inc.status_ga, full.status_ga[rows])
    assert np.array_equal(inc.status_r53, full.status_r53[rows])
    assert np.array_equal(inc.derived, full.derived[rows])


def _device_bytes(torch, ptr, nbytes):
    if not nbytes:
        return np.zeros(0, dtype=np.uint8)

    class _Dev:
        __cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 3}
    return torch.as_tensor(_Dev(), device="cuda").cpu().numpy()


def device_changeset(abi, cs):
    """Host copy of the arrays a gar_diff_device call left on the device, in abi.ChangeSet's form."""
    import torch
    P = lambda p: ctypes.cast(p, ctypes.c_void_p).value  # noqa: E731
    n, n_ops, n_lbi, n_dp = int(cs.n_objects), int(cs.n_ops), int(cs.n_lbi), int(cs.n_dports)
    return SimpleNamespace(
        n_objects=n,
        status_ga=_device_bytes(torch, P(cs.status_ga), 4 * n).view(np.uint32),
        status_r53=_device_bytes(torch, P(cs.status_r53), 4 * n).view(np.uint32),
        derived=_device_bytes(torch, P(cs.derived), 4 * n).view(np.uint32),
        ops=_device_bytes(torch, P(cs.ops), 24 * n_ops).view(abi.OP_DTYPE),
        section_begin=np.array(list(cs.section_begin), dtype=np.uint64),
        tok_code=_device_bytes(torch, P(cs.tok_code), n_lbi),
        tok_name=_device_bytes(torch, P(cs.tok_name), 8 * n_lbi).view(np.uint64),
        tok_region=_device_bytes(torch, P(cs.tok_region), 8 * n_lbi).view(np.uint64),
        dport_begin=_device_bytes(torch, P(cs.dport_begin), 4 * (n + 1)).view(np.uint32),
        dports=_device_bytes(torch, P(cs.dports), 4 * n_dp).view(np.int32))


def assert_same(garecon, got, want, what=""):
    for k in garecon.abi.ChangeSet.ARRAYS:
        a, b = getattr(got, k), getattr(want, k)
        assert a.shape == b.shape and np.array_equal(a, b), (what, k, garecon.abi.ChangeSet.describe_first_mismatch(got, want))


# ------------------------------------------------------------------ full diff, device-resident result

@pytest.mark.parametrize("name", MODELS)
def test_full_diff_eager_recorded_replayed(garecon, engine, models, name):
    """Every full diff on one loaded snapshot equals the oracle: eager, eager on the prepared snapshot, recorded, replayed."""
    m = models(name)
    assert len(m.want.ops) > len(m.objects) // 2
    engine.load(m.snap)
    modes = []
    while not modes or modes[-1] != 2:
        assert len(modes) < 6, modes
        got = engine.diff()
        modes.append(engine.counters()["launch_mode"])
        assert_same(garecon, got, m.want, modes)
    assert 1 in modes


@pytest.mark.parametrize("name", MODELS)
def test_diff_device_contents(garecon, engine, models, name):
    """The arrays gar_diff_device leaves on the device are the gar_diff result byte for byte (the first diff after a load is
    eager, the next ones record and replay: check the device result of each, up to the replayed one)."""
    m = models(name)
    engine.load(m.snap)
    modes = []
    while not modes or modes[-1] != 2:
        assert len(modes) < 6, modes
        cs = engine.diff_device()
        modes.append(engine.counters()["launch_mode"])
        assert_same(garecon, device_changeset(garecon.abi, cs), m.want, modes)
    assert 1 in modes


# ------------------------------------------------------------------ gar_diff_keys

@pytest.mark.parametrize("name", ["rand", "multilbi", "hot"])
def test_diff_keys_batches(garecon, oracle, engine, models, name):
    """Batches of 1 %, 10 % and 100 % of the rows, sorted and shuffled, with deleted keys (rand: the ~4800 dropped objects, whose
    accelerators and records are orphans of the full diff): first call after a load (prepares the snapshot), then a full diff,
    then the batch again on the prepared snapshot.  Equal to the oracle's per-key reconcile and to the full diff's slice."""
    m = models(name)
    for bid, rows in _batches(len(m.objects), MODELS.index(name)):
        engine.load(m.snap)
        before = engine.diff_keys(rows, m.deleted)
        full = engine.diff()
        after = engine.diff_keys(rows, m.deleted)
        want = oracle.diff_keys(m.snap, rows, m.deleted, mode=1)
        assert before.diff(want) == [], (bid, before.describe_first_mismatch(want))
        assert after.diff(want) == [], (bid, after.describe_first_mismatch(want))
        assert full.diff(m.want) == [], (bid, full.describe_first_mismatch(m.want))
        check_against_full(before, full, rows)
    sb = [int(x) for x in want.section_begin]
    assert sb[2] > sb[1] and sb[4] > sb[3]  # the deleted keys own accelerators and records


# ------------------------------------------------------------------ gar_bindings_diff

def test_bindings_diff_at_scale(garecon, oracle, engine, models):
    """10^5 bindings over 4000 endpoint groups (one shared by a fifth of them, 2 % with 64-191 endpoint ids) on a 2*10^4-object
    cluster; the snapshot stays usable for the full diff."""
    m = models("bindings")
    engine.load(m.snap)
    got = engine.bindings_diff(m.bindings)
    want = oracle.bindings_diff(m.snap, m.bindings)
    assert np.array_equal(got.status_ga, want.status_ga)
    assert np.array_equal(got.ops, want.ops), garecon.abi.ChangeSet.describe_first_mismatch(got, want)
    assert len(got.ops) > 1000
    assert_same(garecon, engine.diff(), m.want)


# ------------------------------------------------------------------ engine forms

@pytest.mark.parametrize("form", ["no_tma", "tma_all", "tiny_caps"])
def test_engine_forms(garecon, oracle, monkeypatch, models, form):
    """The 6*10^4-object randmodel cluster with dropped objects, column-major slabs (every staged window holds its block's strings), on
    an engine created with GAR_NO_TMA=1, GAR_TMA_ALL=1 or GAR_TINY_CAPS=1 (every capacity starts at 1: each intermediate
    relation grows and reruns): full diffs through replay and a shuffled 10 % batch equal the oracle."""
    m = models("rand", layout="level")
    if form == "tiny_caps":
        monkeypatch.setenv("GAR_TINY_CAPS", "1")
    rows = _batches(len(m.objects), 7)[3][1]
    want_keys = oracle.diff_keys(m.snap, rows, m.deleted, mode=1)
    with engine_in_form(garecon, monkeypatch, "default" if form == "tiny_caps" else form, cluster_name="default") as e:
        e.load(m.snap)
        modes = []
        for k in range(4):  # eager, eager on the prepared snapshot, recorded, replayed
            assert_same(garecon, e.diff(), m.want, (form, k))
            modes.append(e.counters()["launch_mode"])
        assert modes == [0, 0, 1, 2], (form, modes)
        got = e.diff_keys(rows, m.deleted)
        assert got.diff(want_keys) == [], got.describe_first_mismatch(want_keys)


# ------------------------------------------------------------------ sharded on one GPU

@pytest.mark.parametrize("peers", [False, True], ids=["staged", "peers"])
def test_sharded_eight_ranks(garecon, models, peers):
    """The randmodel cluster with dropped objects cut into 8 slices, rows re-homed through buffers on one GPU (staged) or stored
    straight into the other engines' arenas (peers): the merged result equals the unsharded oracle.  Its bad hostnames put
    hundreds of load balancers under one (name, region) key on one directory shard, where "first row wins" needs the bucket in
    row order (more rows than the per-bucket ordering takes)."""
    m = models("rand")
    if not hasattr(m, "slices"):
        m.slices = [(garecon.pack(objs_r, act_r), sh) for objs_r, act_r, sh in shard.slice_model(m.objects, m.actual, 8)]
    engines, keep = [], []
    try:
        for snap_r, _ in m.slices:
            e = garecon.Engine(cluster_name="default")
            engines.append(e)
            e.load(snap_r)
        if peers:
            shard.exchange_local_peers(engines, [sh for _, sh in m.slices])
        else:
            shard.exchange_local(engines, [sh for _, sh in m.slices], keep, device="cuda:0")
        parts = [e.diff() for e in engines]
    finally:
        for e in engines:
            e.close()
    check_slices(garecon, m.want, parts, len(m.objects))


# ------------------------------------------------------------------ snapshots attached from device buffers

def attach_structs(garecon, snap, slab_offset, keep):
    """Device copies of a packed snapshot's two structs: every column in its own CUDA tensor; each slab at `slab_offset` bytes
    past a 16-byte boundary inside a larger tensor, with SLAB_PAD zero bytes behind it."""
    import torch
    tables = garecon.tables

    def dev(struct, tabs):
        s = type(struct)()
        ctypes.pointer(s)[0] = struct
        for t, (nf, cl) in tabs.items():
            for name, kind in cl:
                arr = tables.columns(struct, {t: (nf, [(name, kind)])})[name]
                x = torch.from_numpy(np.ascontiguousarray(arr).copy() if arr.size else np.zeros(1, dtype=arr.dtype)).cuda()
                keep.append(x)
                setattr(s, name, ctypes.cast(ctypes.c_void_p(x.data_ptr()), type(getattr(s, name))))
        slab = np.ascontiguousarray(tables.columns(struct, {})["slab"])
        buf = torch.zeros(len(slab) + 16 + slab_offset + SLAB_PAD, dtype=torch.uint8, device="cuda")
        start = (-buf.data_ptr()) % 16 + slab_offset
        assert len(buf) - start - len(slab) >= SLAB_PAD
        buf[start:start + len(slab)] = torch.from_numpy(slab).cuda()
        keep.append(buf)
        assert (buf.data_ptr() + start) % 16 == slab_offset
        s.slab = ctypes.cast(ctypes.c_void_p(buf.data_ptr() + start), type(s.slab))
        return s

    o, a = dev(snap.objects, tables.OBJ_TABLES), dev(snap.actual, tables.ACT_TABLES)
    torch.cuda.synchronize()  # the copies run on torch's stream, the engine reads on its own
    return o, a


@pytest.mark.parametrize("slab_offset", [0, 8], ids=["aligned16", "offset8"])
@pytest.mark.parametrize("name,layout", [("rand", "level"), ("bindings", "row")])
def test_attached_snapshot(garecon, oracle, engine, models, name, layout, slab_offset):
    """gar_snapshot_attach_device on caller-owned buffers gives the answers of the loaded snapshot and of the oracle: full
    diff, device-resident result, a shuffled 10 % batch of keys with deleted keys, and bindings.  With slab_offset = 8 the
    slabs are 8-byte aligned only, so every staged row pass takes its direct-load fallback."""
    m = models(name, layout=layout)
    rows = _batches(len(m.objects), 9)[3][1]
    engine.load(m.snap)
    loaded_keys = engine.diff_keys(rows, m.deleted)
    loaded_bindings = engine.bindings_diff(m.bindings) if m.bindings is not None else None
    keep = []
    with garecon.Engine(cluster_name="default") as e:
        e.attach_device(*attach_structs(garecon, m.snap, slab_offset, keep))
        for k in range(4):
            assert_same(garecon, e.diff(), m.want, ("diff", k))
        assert_same(garecon, device_changeset(garecon.abi, e.diff_device()), m.want, "diff_device")
        got = e.diff_keys(rows, m.deleted)
        assert got.diff(loaded_keys) == [], got.describe_first_mismatch(loaded_keys)
        want = oracle.diff_keys(m.snap, rows, m.deleted, mode=1)
        assert got.diff(want) == [], got.describe_first_mismatch(want)
        if m.bindings is not None:
            got = e.bindings_diff(m.bindings)
            assert np.array_equal(got.ops, loaded_bindings.ops) and np.array_equal(got.status_ga, loaded_bindings.status_ga)
            want = oracle.bindings_diff(m.snap, m.bindings)
            assert np.array_equal(got.ops, want.ops) and np.array_equal(got.status_ga, want.status_ga)
        assert_same(garecon, e.diff(), m.want, "diff after the partial entry points")
