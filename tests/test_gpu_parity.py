"""GPU tier: the sm_90a library, called through the C ABI (ctypes), must produce the oracle's change set
bit for bit (integer/index work: no tolerance)."""
import numpy as np
import pytest

import randmodel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", range(24))
def test_random_snapshots_match_oracle(garecon, oracle, engine, seed):
    objects, actual = randmodel.make(seed, n_objects=60)
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    got = engine.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert got.kernel_launches > 0


def test_empty_snapshot(garecon, oracle, engine):
    snap = garecon.pack([], {})
    engine.load(snap)
    got = engine.diff()
    assert got.diff(oracle.diff(snap, "default", mode=1)) == []


def test_objects_without_any_actual_state(garecon, oracle, engine):
    objects, _ = randmodel.make(5, n_objects=50)
    snap = garecon.pack(objects, {})
    engine.load(snap)
    got = engine.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


def test_orphans_only(garecon, oracle, engine):
    """An EMPTY object table while the cluster still owns resources: refused by default (an unsynced informer looks like this,
    include/garecon.h "Orphan sweep precondition"); with allow_empty_cache the orphan sections equal the oracle's."""
    _, actual = randmodel.make(9, n_objects=50)
    snap = garecon.pack([], actual)
    engine.load(snap)
    with pytest.raises(garecon.abi.GarError, match="object table is empty") as ei:
        engine.diff()
    assert ei.value.rc == garecon.abi.GAR_E_STATE
    with garecon.Engine(cluster_name="default", allow_empty_cache=True) as e:
        e.load(snap)
        got = e.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert len(got.ops) > 0


def test_no_orphans_flag_leaves_the_orphan_sections_empty(garecon, oracle):
    """GAR_FLAG_NO_ORPHANS: nothing is deleted on the strength of a key being absent; the object sections are unchanged."""
    objects, actual = randmodel.make(12, n_objects=80)
    snap = garecon.pack(objects[:40], actual)  # half of the objects are gone: their resources are orphans
    want = oracle.diff(snap, "default", mode=1)
    sb = [int(x) for x in want.section_begin]
    assert sb[2] - sb[1] > 0 and sb[4] - sb[3] > 0
    with garecon.Engine(cluster_name="default", orphans=False) as e:
        e.load(snap)
        got = e.diff()
    gb = [int(x) for x in got.section_begin]
    assert gb[2] == gb[1] and gb[4] == gb[3]
    assert np.array_equal(got.ops[gb[0]:gb[1]], want.ops[sb[0]:sb[1]]) and np.array_equal(got.ops[gb[2]:gb[3]], want.ops[sb[2]:sb[3]])
    assert np.array_equal(got.status_ga, want.status_ga) and np.array_equal(got.status_r53, want.status_r53)


def test_golden_hostnames_through_the_abi(garecon, engine):
    """reference load_balancer_test.go:17-40 through the tokeniser kernel."""
    from test_oracle_golden import LB_HOSTNAMES
    objects = [dict(kind="service", ns="default", name=f"s{i}", annotations={}, lb_ingress=[h]) for i, (h, *_r) in enumerate(LB_HOSTNAMES)]
    snap = garecon.pack(objects, {})
    engine.load(snap)
    cs = engine.diff()
    for i, (h, name, region, code) in enumerate(LB_HOSTNAMES):
        assert cs.tok_code[i] == code
        assert snap.obj_str(cs.tok_name[i]).decode() == name
        assert snap.obj_str(cs.tok_region[i]).decode() == region


def test_golden_listen_ports_through_the_abi(garecon, engine):
    """reference global_accelerator_test.go:354-480 + local_e2e fixture through the JSON kernel."""
    anns = ['[{"HTTP": 80}, {"HTTPS": 443}]', '[{"HTTPS":443}]']
    objects = [dict(kind="ingress", ns="default", name=f"i{i}", ingress_class="alb", annotations={"alb.ingress.kubernetes.io/listen-ports": a}, ports=[8080, 80])
               for i, a in enumerate(anns)]
    snap = garecon.pack(objects, {})
    engine.load(snap)
    cs = engine.diff()
    assert list(cs.dport_begin) == [0, 2, 3]
    assert list(cs.dports) == [80, 443, 443]


def test_layout_rule_violation_is_an_error(garecon, engine):
    snap = garecon.pack([dict(kind="service", ns="a", name="b")], {})
    snap.arrays["obj_name"][0] = (1 << garecon.abi.OFF_BITS) | 0  # name no longer follows "ns/"
    with pytest.raises(garecon.GarError) as ei:
        engine.load(snap)
    assert ei.value.rc == garecon.abi.GAR_E_INVALID


def test_bad_string_reference_is_an_error(garecon, engine):
    snap = garecon.pack([dict(kind="service", ns="a", name="b", annotations={"k": "v"})], {})
    snap.arrays["ann_val"][0] = (100 << garecon.abi.OFF_BITS) | 5
    with pytest.raises(garecon.GarError):
        engine.load(snap)


def test_hot_keys_force_the_fallback_paths(garecon, oracle, engine):
    """> 16 duplicates per hash bucket (radix-sort fallback of the index build), > 4 ops per object (re-evaluation
    in the compaction pass), > 8 owned value rows (bucket re-walk): all must stay bit-exact."""
    import hotkeys
    objects, actual = hotkeys.make()
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    got = engine.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert len(got.ops) > 200


def test_tokeniser_fuzz(garecon, oracle, engine):
    import fuzzcases
    snap = garecon.pack(fuzzcases.fuzz_hostnames(12, 5000), {})
    engine.load(snap)
    got = engine.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


def test_listen_ports_fuzz(garecon, oracle, engine):
    import fuzzcases
    snap = garecon.pack(fuzzcases.listen_objects(), {})
    engine.load(snap)
    got = engine.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


def test_huge_value_lists(garecon, oracle, engine):
    """Record sets with > 32 and > 4096 values: the block-wide and grid-wide branches of the record pass."""
    import hotkeys
    objects, actual = hotkeys.make(ndup_acc=3, ndup_alias=2, ndup_val=2100)
    snap = garecon.pack(objects, actual)
    engine.load(snap)
    got = engine.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


@pytest.mark.parametrize("layout", ["level", "reverse", "shuffle"])
def test_results_do_not_depend_on_the_slab_layout(garecon, oracle, engine, layout):
    objects, actual = randmodel.make(17, n_objects=80)
    base = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    snap = garecon.pack(objects, actual, layout=layout, seed=3)
    engine.load(snap)
    got = engine.diff()
    assert got.diff(oracle.diff(snap, "default", mode=1)) == []
    for k in ("status_ga", "status_r53", "derived", "ops", "section_begin", "tok_code", "dport_begin", "dports"):
        assert getattr(got, k).tolist() == getattr(base, k).tolist(), k


def test_capacity_overflow_paths(garecon, oracle, monkeypatch):
    """GAR_TINY_CAPS=1: every capacity starts at 1, so the grow-and-rerun paths of the sync-free pipeline run on the GPU."""
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    for seed in (3, 4):
        objects, actual = randmodel.make(seed, n_objects=200)
        snap = garecon.pack(objects, actual)
        with garecon.Engine(cluster_name="default") as e:
            e.load(snap)
            got = e.diff()
            again = e.diff()
        want = oracle.diff(snap, "default", mode=1)
        assert got.diff(want) == [], got.describe_first_mismatch(want)
        assert again.diff(want) == []


def test_recorded_launch_sequences_replay_the_same_diff(garecon, oracle):
    """The full diff of an unchanged snapshot is recorded into a CUDA graph on its second run and replayed afterwards (engine:
    graph_begin / graph_end).  Replays must reproduce the result; a new snapshot, and the first diff after it, must not see a
    stale recording — with and without GAR_FLAG_REPREPARE."""
    for reprepare in (False, True):
        with garecon.Engine(cluster_name="default", reprepare=reprepare) as e:
            for seed in (31, 32, 31):
                objects, actual = randmodel.make(seed, n_objects=150)
                snap = garecon.pack(objects, actual)
                want = oracle.diff(snap, "default", mode=1)
                e.load(snap)
                for k in range(6):  # eager, eager (prepared), recorded, replayed ...
                    got = e.diff()
                    assert got.diff(want) == [], (reprepare, seed, k, got.describe_first_mismatch(want))
                    assert got.kernel_launches > 0
