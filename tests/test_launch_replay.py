"""Recorded launch sequences (CUDA graphs) replayed after every kind of state change.

The third full diff of an unchanged snapshot is recorded into a CUDA graph and later ones replay it (gar_engine.cu
graph_begin / graph_end).  A replay skips the host side of the pipeline entirely, so it is only right if every call that
changes what the diff reads either drops the recording or leaves the buffers the recording reads as it found them.  The
partial flavours (gar_diff_keys, gar_bindings_diff) write the same scratch slots as the full diff; deltas and loads change the
tables.  Here every operation is followed by full diffs until one is replayed (counters()["launch_mode"] == 2), and every
answer along the way is compared with the oracle on a mirror of the resident snapshot.

The same sequences run on an engine created with GAR_NO_GRAPH=1 (never recorded, identical answers), and on the host
simulation (no graphs at all), which checks the prepared-state bookkeeping (prepared, obj_stale, owners_stale, the on-demand
owner indexes, force_radix, the capacity hints) in the CPU tier."""
import copy
import random

import pytest

import egbcases
import hotkeys
from test_actual_deltas import AwsEvents, AwsModel, apply_delta
from test_object_deltas import Events, Mirror, assert_same_full, key_of

DELETED = [(0, "default/absent-replay-0"), (1, "prod/absent-replay-1")]  # keys in no model: ix_owner / ix_val lookups only
QUERIES = ("keys", "keys_deleted", "bindings", "device", "diff")
MUTATIONS = ("objects", "actual", "refused", "reload", "hot_keys")


class Sequence:
    """One engine, a snapshot and its mirrors (objects: Mirror, AWS tables: AwsModel).  gpu: run full diffs after each operation
    until one is replayed; otherwise (host simulation, GAR_NO_GRAPH=1) run `schedule`'s number of full diffs."""

    def __init__(self, garecon, oracle, engine, seed, n_objects, oracle_mode, gpu, schedule=None):
        self.g, self.oracle, self.e, self.mode, self.gpu = garecon, oracle, engine, oracle_mode, gpu
        objects, actual, bindings, known = egbcases.random_bindings(seed, n_objects=n_objects, n_bindings=3 * n_objects)
        self.b = garecon.pack_bindings(bindings, known)
        self.oev, self.aev = Events(seed, actual), AwsEvents(seed)
        self.rng = random.Random(seed * 17 + 1)
        self.rows = sorted(self.rng.sample(range(n_objects), 8))  # one batch size for every incremental diff: its buffers fit
        self.schedule = list(schedule) if schedule is not None else None
        self.counts, self.results, self.after = [], [], {}
        self._load(objects, actual)

    def _load(self, objects, actual):
        snap = self.snap = self.g.pack(objects, actual)  # the host simulation reads the loaded columns in place
        self.e.load(snap)
        self.om, self.model = Mirror(objects, snap), AwsModel(actual, snap)

    def _msnap(self):
        return self.g.pack(self.om.objects, self.model.actual)

    def launch_mode(self):
        return self.e.counters()["launch_mode"]

    # ---- queries: each answer equals the oracle's; partial diffs report launch mode 0
    def full(self):
        msnap = self._msnap()
        got = self.e.diff()
        assert_same_full(got, self.oracle.diff(msnap, "default", mode=1), self.om.slab, msnap.arrays["o.slab"])
        self.results.append(got)
        return self.launch_mode()

    def keys(self, deleted=()):
        rows = [r for r in self.rows if r < len(self.om.objects)]
        msnap = self._msnap()
        got = self.e.diff_keys(rows, list(deleted))
        want = self.oracle.diff_keys(msnap, rows, list(deleted), mode=self.mode)
        assert got.diff(want) == [], got.describe_first_mismatch(want)
        assert self.launch_mode() == 0

    def bindings(self):
        assert self.e.bindings_diff(self.b).ops.tolist() == self.oracle.bindings_diff(self._msnap(), self.b).ops.tolist()
        assert self.launch_mode() == 0

    def device(self):
        cs = self.e.diff_device()
        want = self.oracle.diff(self._msnap(), "default", mode=1)
        assert int(cs.n_ops) == len(want.ops) and [int(x) for x in cs.section_begin] == [int(x) for x in want.section_begin]

    # ---- state changes
    def objects(self):
        upserts, deleted = self.oev.batch(self.om.objects)
        usnap = self.g.pack(upserts, None) if upserts else None
        res = self.e.apply_objects(usnap.objects if usnap else None, deleted)
        up_row, del_row, _, _ = self.om.apply(upserts, deleted, usnap)
        assert res.upsert_row.tolist() == up_row and res.deleted_row.tolist() == del_row

    def actual(self):
        apply_delta(self.g, self.e, self.model, self.aev.batch(self.model.actual))

    def refused(self):
        with pytest.raises(self.g.GarError) as ei:
            if self.rng.random() < 0.5 and self.om.objects:
                self.e.apply_objects(None, [key_of(self.om.objects[0])] * 2)  # the same key twice
            else:
                self.e.apply_actual(acc_deleted=[0, 0])  # the same row twice (or out of range)
        assert ei.value.rc == self.g.abi.GAR_E_INVALID

    def reload(self):
        """A different snapshot with the same table sizes: load balancer states (or accelerator flags) change, nothing else."""
        actual = copy.deepcopy(self.model.actual)
        lbs, accs = actual.get("lbs", []), actual.get("accelerators", [])
        for lb in lbs:
            lb["state"] = self.rng.choice(["active", "provisioning", "failed", "active_impaired"])
        if not lbs:
            for a in accs:
                a["enabled"] = not a.get("enabled", True)
        self._load(list(self.om.objects), actual)

    def hot_keys(self):
        """More duplicates per hash bucket than the per-bucket ordering takes: the load's first diff rebuilds with force_radix."""
        objects, actual = hotkeys.make()
        self._load(objects, actual)

    def settle(self, op):
        """Full diffs after `op`: until one is replayed (GPU), or as many as the GPU run needed.  -> their launch modes."""
        if self.schedule is not None:
            modes = [self.full() for _ in range(self.schedule.pop(0))]
        elif self.gpu:
            modes = []
            while not modes or modes[-1] != 2:
                assert len(modes) < 6, (op, modes)
                modes.append(self.full())
            assert modes == [2] or modes == [0] * (len(modes) - 2) + [1, 2], (op, modes)
        else:
            modes = [self.full() for _ in range(2)]
        self.counts.append(len(modes))
        self.after.setdefault(op, []).append(modes)
        return modes

    def run(self, op):
        if op == "keys":
            self.keys()
        elif op == "keys_deleted":
            self.keys(DELETED)
        elif op != "diff":
            getattr(self, op)()
        return self.settle(op)

    def warm(self):
        """Every flavour once at its batch size: later calls reuse their buffers, so none of them drops the recording."""
        self.keys()
        self.keys(DELETED)  # the first deleted key builds ix_owner / ix_val
        self.bindings()
        self.device()


def scripted(seq):
    seq.warm()
    seq.settle("load")
    for op in QUERIES:
        modes = seq.run(op)
        if seq.gpu and seq.schedule is None:
            assert modes[0] == 2, (op, modes)  # the diff right after a query replays the recording
    for op in MUTATIONS:
        seq.run(op)
        seq.warm()
        seq.settle(op + "+warm")
    return seq


def random_ops(seq, seed, n_ops=14):
    rng = random.Random(seed)
    seq.warm()
    seq.settle("load")
    ops = list(QUERIES + MUTATIONS) + [rng.choice(QUERIES + MUTATIONS[:3]) for _ in range(n_ops - len(QUERIES + MUTATIONS))]
    rng.shuffle(ops)
    for op in ops:
        seq.run(op)
        if op in MUTATIONS:  # new table sizes: the next queries' buffers are sized once, outside the checked step
            seq.warm()
            seq.settle(op + "+warm")
    return seq


def _engine(garecon, monkeypatch, no_graph):
    monkeypatch.delenv("GAR_NO_GRAPH", raising=False)
    if no_graph:
        monkeypatch.setenv("GAR_NO_GRAPH", "1")
    return garecon.Engine(cluster_name="default")


def _same_results(a, b):
    assert len(a.results) == len(b.results)
    for k, (x, y) in enumerate(zip(a.results, b.results)):
        assert x.diff(y) == [], (k, x.describe_first_mismatch(y))


@pytest.fixture(scope="module")
def hostlib(garecon):
    import __graft_entry__ as ge
    return garecon.abi.load_library(ge.build_hostsim())


# ------------------------------------------------------------------ host simulation

def test_hostsim_scripted_sequence(garecon, oracle, hostlib):
    with garecon.Engine(cluster_name="default", lib=hostlib) as e:
        seq = scripted(Sequence(garecon, oracle, e, 3, 60, 0, gpu=False))
    assert {m for ms in seq.after.values() for modes in ms for m in modes} == {0}


@pytest.mark.parametrize("seed", range(6))
def test_hostsim_random_sequences(garecon, oracle, hostlib, seed):
    with garecon.Engine(cluster_name="default", lib=hostlib) as e:
        seq = random_ops(Sequence(garecon, oracle, e, seed, 60, 0, gpu=False), seed)
    assert {m for ms in seq.after.values() for modes in ms for m in modes} == {0}


# ------------------------------------------------------------------ GPU

@pytest.mark.gpu
def test_gpu_scripted_sequence(garecon, oracle, monkeypatch):
    with _engine(garecon, monkeypatch, False) as e:
        seq = scripted(Sequence(garecon, oracle, e, 3, 80, 1, gpu=True))
    for op in MUTATIONS:
        assert seq.after[op][0][0] == 0, op  # the recording of the old state is never replayed
    with _engine(garecon, monkeypatch, True) as e:
        ctl = scripted(Sequence(garecon, oracle, e, 3, 80, 1, gpu=True, schedule=seq.counts))
    assert {m for ms in ctl.after.values() for modes in ms for m in modes} == {0}
    _same_results(seq, ctl)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(6))
def test_gpu_random_sequences(garecon, oracle, monkeypatch, seed):
    with _engine(garecon, monkeypatch, False) as e:
        seq = random_ops(Sequence(garecon, oracle, e, seed, 80, 1, gpu=True), seed)
    for op in QUERIES + MUTATIONS:
        assert any(modes[-1] == 2 for modes in seq.after[op]), op
    for op in ("keys", "keys_deleted", "bindings", "device", "diff"):
        assert any(modes[0] == 2 for modes in seq.after[op]), (op, seq.after[op])
    with _engine(garecon, monkeypatch, True) as e:
        ctl = random_ops(Sequence(garecon, oracle, e, seed, 80, 1, gpu=True, schedule=seq.counts), seed)
    assert {m for ms in ctl.after.values() for modes in ms for m in modes} == {0}
    _same_results(seq, ctl)
