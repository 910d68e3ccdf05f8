"""GPU tier at BASELINE sizes: bit-exact against the indexed oracle (itself proven equal to the faithful
restatement at small sizes in test_synth_configs.py), plus size-independent properties of the change set."""
import importlib
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def synth(garecon):
    import __graft_entry__ as ge
    ge.build_synth()
    return importlib.import_module("aws-global-accelerator-controller_b200.synth")


def _check_properties(cs, snap):
    sb = cs.section_begin.astype(np.int64)
    assert sb[0] == 0 and (np.diff(sb) >= 0).all() and sb[-1] == len(cs.ops)
    ops = cs.ops
    for s in (0, 2):  # object sections are ordered by object row
        part = ops[sb[s]:sb[s + 1]]
        assert (np.diff(part["obj"].astype(np.int64)) >= 0).all()
    assert (ops[sb[1]:sb[2]]["obj"] == 0xFFFFFFFF).all() and (ops[sb[3]:sb[4]]["obj"] == 0xFFFFFFFF).all()
    ga = ops[sb[1]:sb[2]]
    assert (np.diff(ga["a0"].astype(np.int64)) > 0).all()  # GA orphans: strictly ascending accelerator rows
    r53o = ops[sb[3]:sb[4]]
    key = r53o["a0"].astype(np.int64) * 2 + r53o["sub"]
    assert (np.diff(key) >= 0).all()  # R53 orphans: (zone, phase) ascending
    codes = ops["head"] & 0xFF
    assert ((codes >= 1) & (codes <= 10)).all()
    ctrl = (ops["head"] >> 8) & 0xFF
    assert (ctrl[:sb[2]] == 0).all() and (ctrl[sb[2]:] == 1).all()
    # ignored objects never produce ops; every op's object is eligible
    st_ga = cs.status_ga & 0xFF
    objs = ops[sb[0]:sb[1]]["obj"]
    assert (st_ga[objs] != 0).all()


@pytest.mark.parametrize("cfg,n", [(2, 100_000), (3, 100_000), (5, 100_000)])
def test_baseline_configs_1e5_bit_exact(garecon, oracle, engine, synth, cfg, n):
    snap = synth.generate(cfg, n)
    engine.load(snap)
    got = engine.diff()
    want = oracle.diff(snap, "default", mode=1, threads=os.cpu_count() or 4)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    _check_properties(got, snap)


@pytest.mark.parametrize("cfg,form", [pytest.param(3, "default", id="3"), pytest.param(5, "default", id="5"),
                                      pytest.param(3, "no_tma", id="3-no_tma"), pytest.param(3, "tma_all", id="3-tma_all")])
def test_column_major_slabs_1e5_bit_exact(garecon, oracle, engine, synth, monkeypatch, cfg, form):
    """bench.py's default input layout (every string column contiguous, as host/packer.hpp writes it): same change set as the
    row-major layout of the same cluster, and equal to the oracle on it.  Config 3 also runs on engines created with
    GAR_NO_TMA=1 (every staged row pass in its direct-load form) and GAR_TMA_ALL=1 (every one staged)."""
    from test_backend_kernels import engine_in_form
    snap = synth.generate(cfg, 100_000, layout=1)
    if form != "default":
        with engine_in_form(garecon, monkeypatch, form, cluster_name=snap.cluster) as e:
            e.load(snap)
            got = e.diff()
    else:
        engine.load(snap)
        got = engine.diff()
    want = oracle.diff(snap, snap.cluster, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    row = synth.generate(cfg, 100_000)
    engine.load(row)
    base = engine.diff()
    for k in ("status_ga", "status_r53", "derived", "ops", "section_begin", "tok_code", "dports"):
        assert np.array_equal(getattr(got, k), getattr(base, k)), k


def test_config3_1e6_bit_exact_and_idempotent(garecon, oracle, engine, synth):
    """BASELINE configs[2] at full size (the bench workload)."""
    snap = synth.generate(3, 1_000_000)
    engine.load(snap)
    got = engine.diff()
    again = engine.diff()
    assert got.diff(again) == []  # a diff does not disturb the loaded snapshot
    _check_properties(got, snap)
    want = oracle.diff(snap, "default", mode=1, threads=os.cpu_count() or 4)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert got.checksum() == want.checksum()


def test_bench_workload_1e6_column_major_bit_exact(garecon, oracle, engine, synth):
    """The exact workload bench.py times on rank 0 (configs[2], 10^6 objects, the preset's seed, COLUMN-major slabs) against the
    oracle — bench.py repeats this comparison inside every run (`parity` in its JSON line)."""
    cfg = synth.preset(3, 1_000_000)
    cfg.layout = 1
    snap = synth.SynthSnapshot(cfg)
    engine.load(snap)
    got = engine.diff()
    _check_properties(got, snap)
    want = oracle.diff(snap, snap.cluster, mode=1, threads=os.cpu_count() or 4)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert got.checksum() == want.checksum()


def _mem_available_gb():
    try:
        for line in open("/proc/meminfo"):
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 1e6
    except OSError:
        pass
    return 0.0


def test_config4_1e7_single_gpu_bit_exact(garecon, oracle, synth):
    """BASELINE configs[3] at its full size on ONE GPU: the 10^7-object cluster bench.py shards across GPUs (generator preset 4,
    16 chunks, column-major slabs), diffed unsharded and compared bit for bit with the oracle on all host cores.  This pins the
    single-GPU result that the sharded runs are checksum-compared with (bench.py `sharded.checksum_equal`)."""
    if _mem_available_gb() < 120:
        pytest.skip("needs ~100 GB of host memory for the 10^7-object tables, the oracle's indexes and two change sets")
    shard = importlib.import_module("aws-global-accelerator-controller_b200.shard")
    n = 10_000_000
    slices = synth.cluster_slices(4, n, 1, layout=1, n_chunks=16, threads=min(32, os.cpu_count() or 4))
    union = garecon.tables.concat_slices(slices)
    del slices
    assert union.objects.n_objects == n
    with garecon.Engine(cluster_name="default", reprepare=True) as e:
        e.load(union)
        got = e.diff()
    _check_properties(got, union)
    want = oracle.diff(union, "default", mode=1, threads=os.cpu_count() or 4)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert shard.canonical_checksum(got) == shard.canonical_checksum(want)
    assert len(got.ops) > n // 4


def test_adversarial_1e6_properties_and_sampled_parity(garecon, oracle, engine, synth):
    """BASELINE configs[4]: 90% colliding hostnames + 64-port listeners at 10^6; full oracle comparison."""
    snap = synth.generate(5, 1_000_000)
    engine.load(snap)
    got = engine.diff()
    _check_properties(got, snap)
    want = oracle.diff(snap, "default", mode=1, threads=os.cpu_count() or 4)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


def test_device_resident_path_matches_host_path(garecon, engine, synth):
    snap = synth.generate(2, 50_000)
    engine.load(snap)
    full = engine.diff()
    cs = engine.diff_device()
    assert int(cs.n_ops) == len(full.ops)
    assert list(cs.section_begin) == list(full.section_begin)
    # the second diff reuses the prepared snapshot (digests + indexes stay resident): fewer launches, same result
    assert 0 < cs.kernel_launches < full.kernel_launches


def test_reprepare_flag_runs_the_complete_pipeline_every_time(garecon, synth):
    snap = synth.generate(2, 20_000)
    with garecon.Engine(cluster_name="default", reprepare=True) as e:
        e.load(snap)
        a = e.diff()
        b = e.diff()
    assert a.diff(b) == []
    assert a.kernel_launches == b.kernel_launches


@pytest.mark.parametrize("cfg", [2, 3, 5])
def test_no_performance_cliff(garecon, synth, cfg):
    """Not a benchmark: a loose bound that catches algorithmic cliffs (a per-record loop over a 10^5-value hot TXT set once
    cost 70x on config 5).  At 10^6 objects a complete diff takes 3-5 ms; allow 10x."""
    snap = synth.generate(cfg, 1_000_000)
    with garecon.Engine(cluster_name=snap.cluster, reprepare=True) as e:
        e.load(snap)
        e.diff_device()
        ms = min(e.diff_device().ms_kernels for _ in range(3))
    assert ms < 50.0, f"config {cfg}: {ms:.1f} ms for 10^6 objects"
