"""Incremental mode (gar_diff_keys; SURVEY.md §8 row f4): the decisions for a batch of work-queue keys — object rows whose
events fired + keys that left the cache — must equal per-key reconciles (oracle), and, for the rows, the slice of the
full diff that belongs to them."""
import random

import numpy as np
import pytest

import randmodel
import scalemodels


def _pick(objects, actual, rng):
    n = len(objects)
    rows = sorted(rng.sample(range(n), k=min(n, rng.randrange(0, n + 1))))
    if rng.random() < 0.3:
        rng.shuffle(rows)  # the order of the batch is the caller's; results follow it
    deleted = []
    owners = []
    for acc in actual.get("accelerators", []):
        owners.append(dict(acc["tags"]).get("aws-global-accelerator-owner", ""))
    for z in actual.get("zones", []):
        for r in z.get("records", []):
            for v in r.get("values", []):
                if v.startswith('"heritage=') and v.count(",") >= 2:
                    owners.append(v.rsplit(",", 1)[1].rstrip('"'))
    for ow in rng.sample(owners, k=min(len(owners), 8)):
        parts = ow.split("/")
        if len(parts) == 3 and parts[0] in ("service", "ingress"):
            deleted.append((0 if parts[0] == "service" else 1, parts[1] + "/" + parts[2]))
    deleted.append((0, "default/never-existed"))
    deleted.append((1, "no-slash"))
    return rows, deleted


def _check_against_full(inc, full, rows):
    """Object-section ops of the incremental result == the full diff's ops for those rows, in batch order."""
    sb = [int(x) for x in full.section_begin]
    for sec, isec in ((0, 0), (2, 2)):
        fops = full.ops[sb[sec]:sb[sec + 1]]
        want = []
        for r in rows:
            want.extend(tuple(int(x) for x in op) for op in fops[fops["obj"] == r].tolist())
        isb = [int(x) for x in inc.section_begin]
        got = [tuple(int(x) for x in op) for op in inc.ops[isb[isec]:isb[isec + 1]].tolist()]
        assert got == want
    assert list(inc.status_ga) == [int(full.status_ga[r]) for r in rows]
    assert list(inc.status_r53) == [int(full.status_r53[r]) for r in rows]
    assert list(inc.derived) == [int(full.derived[r]) for r in rows]


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


@pytest.mark.parametrize("seed", range(20))
def test_hostsim_keys_match_oracle_and_full_diff(garecon, oracle, hostsim, seed):
    rng = random.Random(seed)
    objects, actual = randmodel.make(seed, n_objects=40)
    snap = garecon.pack(objects, actual)
    rows, deleted = _pick(objects, actual, rng)
    hostsim.load(snap)
    inc = hostsim.diff_keys(rows, deleted)       # first call after a load prepares the snapshot
    full = hostsim.diff()                         # full diff on the already prepared snapshot
    inc2 = hostsim.diff_keys(rows, deleted)      # and again, now fully cached
    want = oracle.diff_keys(snap, rows, deleted, mode=0)
    assert inc.diff(want) == [], inc.describe_first_mismatch(want)
    assert inc2.diff(want) == []
    assert full.diff(oracle.diff(snap, "default", mode=1)) == []
    _check_against_full(inc, full, rows)


def test_hostsim_dropped_objects(garecon, oracle, hostsim):
    """A 2000-object randmodel cluster with 8 % of its objects dropped after generation: their accelerators, TXT owner values and
    alias records are orphans (randmodel alone makes 0-3 at any size).  Full diff, and a shuffled 10 % batch with the dropped
    keys (and keys that match nothing) as deleted keys."""
    objects, actual, dropped = scalemodels.randmodel_dropped(2, 2000)
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    full = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert full.diff(want) == [], full.describe_first_mismatch(want)
    sb = [int(x) for x in want.section_begin]
    assert len(dropped) > 100 and sb[2] - sb[1] > 50 and sb[4] - sb[3] > 200
    rows = random.Random(2).sample(range(len(objects)), len(objects) // 10)
    deleted = dropped + scalemodels.ABSENT_KEYS
    inc = hostsim.diff_keys(rows, deleted)
    want = oracle.diff_keys(snap, rows, deleted, mode=1)
    assert inc.diff(want) == [], inc.describe_first_mismatch(want)
    _check_against_full(inc, full, rows)


def test_hostsim_empty_batch(garecon, oracle, hostsim):
    objects, actual = randmodel.make(1, n_objects=20)
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    inc = hostsim.diff_keys([], [])
    assert len(inc.ops) == 0 and inc.n_objects == 0


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(300, 312))
def test_gpu_keys_match_oracle_and_full_diff(garecon, oracle, engine, seed):
    rng = random.Random(seed)
    objects, actual = randmodel.make(seed, n_objects=90)
    snap = garecon.pack(objects, actual)
    rows, deleted = _pick(objects, actual, rng)
    engine.load(snap)
    inc = engine.diff_keys(rows, deleted)
    full = engine.diff()
    inc2 = engine.diff_keys(rows, deleted)
    want = oracle.diff_keys(snap, rows, deleted, mode=1)
    assert inc.diff(want) == [], inc.describe_first_mismatch(want)
    assert inc2.diff(want) == []
    _check_against_full(inc, full, rows)


@pytest.mark.gpu
def test_gpu_keys_at_scale(garecon, oracle, engine):
    """10^5-object cluster, a 1 % batch of dirty keys: same decisions as the full diff, a fraction of the work."""
    import importlib
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    snap = synth.generate(3, 100_000)
    engine.load(snap)
    full = engine.diff()
    rng = random.Random(1)
    rows = sorted(rng.sample(range(100_000), 1000))
    inc = engine.diff_keys(rows, [])
    _check_against_full(inc, full, rows)
    want = oracle.diff_keys(snap, rows, [], mode=1)
    assert inc.diff(want) == [], inc.describe_first_mismatch(want)
    assert inc.kernel_launches < full.kernel_launches
