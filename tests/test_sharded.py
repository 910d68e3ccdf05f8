"""Sharded mode (SURVEY.md §8 row e, BASELINE configs[3]): one cluster cut into n_ranks slices, rows re-homed by key hash in
two exchanges, every shard running the ordinary pipeline on its self-contained sub-snapshot.  The merged result must equal
the unsharded change set of the whole cluster bit for bit (oracle on the concatenated model).

CPU tier: the device code compiled for the host (tests/hostsim), all ranks' engines in one process; a 2-process gloo test
covers the torch.distributed data path (tests/test_ranks_gloo.py style)."""
import importlib

import numpy as np
import pytest

import hotkeys
import randmodel

shard = importlib.import_module("aws-global-accelerator-controller_b200.shard")


@pytest.fixture(scope="module")
def hostlib(garecon):
    import __graft_entry__ as ge
    return garecon.abi.load_library(ge.build_hostsim())


def run_sharded(garecon, lib, objects, actual, n_ranks, cluster="default"):
    slices = shard.slice_model(objects, actual, n_ranks)
    engines, snaps, keep = [], [], []
    for objs_r, act_r, _ in slices:
        e = garecon.Engine(cluster_name=cluster, lib=lib)
        snap = garecon.pack(objs_r, act_r)
        e.load(snap)
        engines.append(e)
        snaps.append(snap)
    shard.exchange_local(engines, [s[2] for s in slices], keep)
    parts = [e.diff() for e in engines]
    for e in engines:
        e.close()
    return shard.merge_changesets(parts, len(objects)), parts


def check(garecon, oracle, lib, objects, actual, n_ranks, cluster="default"):
    got, parts = run_sharded(garecon, lib, objects, actual, n_ranks, cluster)
    want = oracle.diff(garecon.pack(objects, actual), cluster, mode=1)
    assert np.array_equal(got["status_ga"], want.status_ga), first_diff(got["status_ga"], want.status_ga)
    assert np.array_equal(got["status_r53"], want.status_r53), first_diff(got["status_r53"], want.status_r53)
    assert np.array_equal(got["derived"], want.derived)
    assert got["section_begin"].tolist() == want.section_begin.tolist()
    assert got["ops"].tolist() == want.ops.tolist(), first_diff(got["ops"].tolist(), want.ops.tolist())
    return got, parts


def first_diff(a, b):
    for i, (x, y) in enumerate(zip(a, b)):
        if x != y:
            return f"first difference at {i}: {x} vs {y}"
    return f"lengths {len(a)} vs {len(b)}"


@pytest.mark.parametrize("n_ranks", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("seed", range(6))
def test_sharded_matches_unsharded(garecon, oracle, hostlib, seed, n_ranks):
    objects, actual = randmodel.make(seed, n_objects=60)
    check(garecon, oracle, hostlib, objects, actual, n_ranks)


@pytest.mark.parametrize("seed,n_ranks", [(40, 2), (41, 3), (42, 8)])
def test_sharded_copy_merge_fallback(garecon, oracle, hostlib, seed, n_ranks, monkeypatch):
    """By default the merged sub-snapshot's strings stay in the receive buffers (no byte is copied); when the two rounds' buffers
    lie further apart than a string offset reaches the engine copies them into merged slabs instead.  Same results."""
    monkeypatch.setenv("GAR_SHARD_COPY_MERGE", "1")
    objects, actual = randmodel.make(seed, n_objects=60)
    check(garecon, oracle, hostlib, objects, actual, n_ranks)


@pytest.mark.parametrize("seed", range(6, 30))
def test_sharded_more_seeds(garecon, oracle, hostlib, seed):
    objects, actual = randmodel.make(seed, n_objects=40)
    check(garecon, oracle, hostlib, objects, actual, 2 + seed % 3)


@pytest.mark.parametrize("seed", range(6))
def test_sharded_multi_lbingress_models(garecon, oracle, hostlib, seed):
    """Self-observation ops carry GAR_PENDING arguments: they must survive the local -> global row translation of a shard."""
    import multilbi
    objects, actual = multilbi.make(seed, n_objects=40)
    got, _ = check(garecon, oracle, hostlib, objects, actual, 2 + seed % 3)
    assert any(0xFFFFFFFE in (int(o["a0"]), int(o["a1"]), int(o["a2"])) for o in got["ops"])


@pytest.mark.parametrize("seed,n_ranks", [(0, 2), (1, 3), (2, 4), (3, 8), (4, 1)])
def test_peer_memory_exchange_matches_unsharded(garecon, oracle, hostlib, seed, n_ranks):
    """include/garecon.h "Peer-memory exchange": every rank's pack stores straight into the other ranks' receive arenas at the
    offsets all ranks derive from the gathered meta rows — same sub-snapshots, same merged result as the all-to-all path."""
    objects, actual = randmodel.make(seed, n_objects=60)
    slices = shard.slice_model(objects, actual, n_ranks)
    engines, snaps = [], []
    for objs_r, act_r, _ in slices:
        e = garecon.Engine(cluster_name="default", lib=hostlib)
        snap = garecon.pack(objs_r, act_r)
        e.load(snap)
        engines.append(e)
        snaps.append(snap)
    shard.exchange_local_peers(engines, [s[2] for s in slices])
    parts = [e.diff() for e in engines]
    for e in engines:
        e.close()
    got = shard.merge_changesets(parts, len(objects))
    want = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    assert np.array_equal(got["status_ga"], want.status_ga) and np.array_equal(got["status_r53"], want.status_r53)
    assert got["ops"].tolist() == want.ops.tolist(), first_diff(got["ops"].tolist(), want.ops.tolist())


def test_sharded_hot_keys(garecon, oracle, hostlib):
    """Many owners claim the same record names / hostnames: alias records replicate to several homes, directory shards see
    long duplicate chains."""
    objects, actual = hotkeys.make()
    got, parts = check(garecon, oracle, hostlib, objects, actual, 4)
    assert len(got["ops"]) > 200
    assert sum(p.n_objects for p in parts) == len(objects)


def long_string_model():
    ANN = "aws-global-accelerator-controller.h3poteto.dev/"
    M, O, H, C = ("aws-global-accelerator-controller-managed", "aws-global-accelerator-owner", "aws-global-accelerator-target-hostname", "aws-global-accelerator-cluster")
    objects, lbs, accs, want_update = [], [], [], []
    for k in range(14):
        lbname = f"{k:032x}"
        host = f"{lbname}-0123456789abcdef.elb.us-west-2.amazonaws.com"
        long_v = "".join(chr(65 + (i * 5 + k) % 26) for i in range(3001 + 17 * k))
        ann = {ANN + "global-accelerator-managed": "true", "service.beta.kubernetes.io/aws-load-balancer-type": "nlb", ANN + "global-accelerator-tags": "k=" + long_v,
               "example.com/blob": "".join(chr(97 + (i * 7 + k) % 26) for i in range(5000 + 13 * k))}
        objects.append(dict(kind="service", ns="default", name=f"s{k}", spec_type="LoadBalancer", annotations=ann, ports=[(80, "TCP")], lb_ingress=[host]))
        lbs.append({"region": "us-west-2", "name": lbname, "dns": host, "arn": f"arn:lb{k}", "state": "active"})
        off = k % 2 == 1
        want_update.append(off)
        accs.append({"arn": f"a{k}", "name": f"service-default-s{k}", "dns": f"a{k}.awsglobalaccelerator.com", "enabled": True,
                     "tags": [(M, "true"), (O, f"service/default/s{k}"), (H, host), (C, "default"), ("k", long_v[:-1] + "!" if off else long_v)],
                     "listeners": [{"arn": f"l{k}", "proto": "TCP", "ports": [80], "egs": [{"arn": f"e{k}", "endpoints": [f"arn:lb{k}"]}]}]})
    return objects, {"lbs": lbs, "accelerators": accs, "zones": []}, want_update


def test_sharded_long_strings(garecon, oracle, hostlib):
    """Strings longer than the pack kernel's per-thread cut (2 KB) are finished by the strided second pass; every byte must
    arrive: a Service whose 3 KB user tag is already on its accelerator needs no op, one whose LAST byte differs needs an update."""
    objects, actual, want_update = long_string_model()
    for n_ranks in (2, 3):
        got, _ = check(garecon, oracle, hostlib, objects, actual, n_ranks)
        sb = [int(x) for x in got["section_begin"]]
        ops = got["ops"][sb[0]:sb[1]]
        assert [int(o["obj"]) for o in ops] == [k for k in range(14) if want_update[k]]
        assert all(int(o["head"]) & 0xFF == 2 for o in ops)  # GA_UPDATE_ACCEL


def test_sharded_other_cluster_name(garecon, oracle, hostlib):
    objects, actual = randmodel.make(3, n_objects=40, cluster="prod-1")
    check(garecon, oracle, hostlib, objects, actual, 3, cluster="prod-1")


def test_sharded_empty_and_lopsided(garecon, oracle, hostlib):
    check(garecon, oracle, hostlib, [], {}, 2)
    objects, actual = randmodel.make(11, n_objects=5)  # fewer objects than ranks: some slices are empty
    check(garecon, oracle, hostlib, objects, actual, 8)
    check(garecon, oracle, hostlib, objects, {}, 3)
    check(garecon, oracle, hostlib, [], actual, 3)


def test_diff_in_the_middle_of_a_new_exchange_is_refused(garecon, hostlib):
    """The sub-snapshot's strings stay in the receive buffers (no copy): once the next exchange has started they are being
    refilled, so a diff must wait for both rounds — GAR_E_STATE instead of decisions about half-overwritten strings."""
    objects, actual = randmodel.make(7, n_objects=40)
    slices = shard.slice_model(objects, actual, 2)
    engines, keep, snaps = [], [], []
    for objs_r, act_r, _ in slices:
        e = garecon.Engine(cluster_name="default", lib=hostlib)
        snaps.append(garecon.pack(objs_r, act_r))
        e.load(snaps[-1])
        engines.append(e)
    shards = [s[2] for s in slices]
    assert engines[0].diff().n_objects == len(slices[0][0])  # before any exchange: the slice itself is diffed
    shard.exchange_local(engines, shards, keep)
    first = [e.diff() for e in engines]
    engines[0].shard_route(shards[0], 1)                     # a new exchange starts on rank 0 ...
    with pytest.raises(garecon.abi.GarError) as ei:
        engines[0].diff()                                    # ... its old sub-snapshot is no longer readable
    assert ei.value.rc == garecon.abi.GAR_E_STATE
    engines[1].shard_route(shards[1], 1)
    keep2 = []
    # finish the exchange properly (route is idempotent: exchange_local routes again) and compare with the first result
    shard.exchange_local(engines, shards, keep2)
    second = [e.diff() for e in engines]
    for a, b in zip(first, second):
        assert a.ops.tolist() == b.ops.tolist() and a.status_ga.tolist() == b.status_ga.tolist()
    for e in engines:
        e.close()


def test_contract_violations_are_errors(garecon, hostlib):
    """The two layout rules of sharded mode are checked on the device: same zone table everywhere, whole zones per rank in
    ascending ranges."""
    objects, actual = randmodel.make(2, n_objects=40)
    slices = shard.slice_model(objects, actual, 2)

    def run(mutate):
        engines, keep = [], []
        for r, (objs_r, act_r, _) in enumerate(slices):
            act_r = mutate(r, act_r)
            e = garecon.Engine(cluster_name="default", lib=hostlib)
            snap = garecon.pack(objs_r, act_r)
            keep.append(snap)
            e.load(snap)
            engines.append(e)
        try:
            shard.exchange_local(engines, [s[2] for s in slices], keep)
        finally:
            for e in engines:
                e.close()

    def rename_zone(r, act):
        if r == 1 and act["zones"]:
            act = dict(act, zones=[dict(act["zones"][0], name="other.example.org.")] + act["zones"][1:])
        return act

    def swap_records(r, act):  # rank 0 holds the LAST zones' records, rank 1 the first ones': ranges descend with the rank
        other = slices[1 - r][1]["zones"]
        return dict(act, zones=[dict(z, records=other[i]["records"]) for i, z in enumerate(act["zones"])])

    assert sum(len(z["records"]) for z in slices[0][1]["zones"]) > 0 and sum(len(z["records"]) for z in slices[1][1]["zones"]) > 0
    with pytest.raises(garecon.abi.GarError, match="zone table"):
        run(rename_zone)
    with pytest.raises(garecon.abi.GarError, match="whole zones"):
        run(swap_records)
    run(lambda r, act: act)  # the unmodified slices are fine


def test_shards_are_balanced_and_disjoint(garecon, oracle, hostlib):
    objects, actual = randmodel.make(5, n_objects=400)
    got, parts = check(garecon, oracle, hostlib, objects, actual, 4)
    sizes = [p.n_objects for p in parts]
    assert sum(sizes) == 400 and min(sizes) > 50


# ------------------------------------------------------------------ generator slices (the bench workload of configs[3])

def run_sharded_slices(garecon, lib, slices, device="cpu", peers=False, **engine_kw):
    tables = garecon.tables
    bases = tables.shard_bases(slices)
    engines, keep = [], []
    for o, a in slices:
        e = garecon.Engine(cluster_name="default", lib=lib, **engine_kw)
        snap = tables.from_columns(o, a)
        e.load(snap)
        engines.append(e)
        keep.append(snap)  # hostsim reads the columns in place
    if peers:
        shard.exchange_local_peers(engines, bases)
    else:
        shard.exchange_local(engines, bases, keep, device=device)
    parts = [e.diff() for e in engines]
    for e in engines:
        e.close()
    return parts


def check_slices(garecon, want, parts, n_total):
    got = shard.merge_changesets(parts, n_total)
    assert np.array_equal(got["status_ga"], want.status_ga)
    assert np.array_equal(got["status_r53"], want.status_r53)
    assert np.array_equal(got["derived"], want.derived)
    assert got["section_begin"].tolist() == want.section_begin.tolist()
    assert np.array_equal(got["ops"], want.ops), first_diff(got["ops"].tolist(), want.ops.tolist())


@pytest.mark.parametrize("cfg,n_total,n_ranks,layout,n_chunks", [(4, 1500, 3, 0, None), (5, 1200, 4, 0, None), (3, 1000, 2, 0, None), (4, 1200, 3, 1, None),
                                                                 (4, 1600, 2, 1, 8), (4, 1600, 4, 1, 8)])
def test_generator_slices_on_hostsim(garecon, oracle, hostlib, cfg, n_total, n_ranks, layout, n_chunks):
    """Chunked generator output (objects / accelerators / LBs of different chunks on one rank) == the union, via the oracle;
    also with column-major string slabs in the slices, and with several generator chunks per rank (bench.py's 10^7 cluster is
    16 chunks whatever the number of GPUs)."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    slices = synth.cluster_slices(cfg, n_total, n_ranks, layout=layout, n_chunks=n_chunks, threads=4)
    union = garecon.tables.concat_slices(slices)
    assert union.objects.n_objects == n_total
    want = oracle.diff(union, "default", mode=1)
    parts = run_sharded_slices(garecon, hostlib, slices)
    check_slices(garecon, want, parts, n_total)
    assert len(want.ops) > n_total // 4
    # the merge-free checksum bench.py uses at 10^7 objects: adds over the shards to the unsharded value
    assert shard.add_checksums([shard.canonical_checksum(p) for p in parts]) == shard.canonical_checksum(want)


def test_canonical_checksum_is_sensitive(garecon, oracle):
    """The additive checksum notices a changed status word, a changed op field, two ops of one object swapped, and an op moved
    to another section boundary."""
    import copy
    objects, actual = randmodel.make(4, n_objects=120)
    cs = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    base = shard.canonical_checksum(cs)
    assert base == shard.canonical_checksum(copy.deepcopy(cs))
    x = copy.deepcopy(cs)
    x.status_r53[7] ^= 0x100
    assert shard.canonical_checksum(x) != base
    x = copy.deepcopy(cs)
    x.ops["a1"][3] ^= 1
    assert shard.canonical_checksum(x) != base
    sb = [int(v) for v in cs.section_begin]
    objs = cs.ops["obj"][sb[0]:sb[1]]
    same = [k for k in range(len(objs) - 1) if objs[k] == objs[k + 1] and cs.ops[k] != cs.ops[k + 1]]
    assert same, "the model should contain an object with two different GA ops"
    x = copy.deepcopy(cs)
    x.ops[[same[0], same[0] + 1]] = x.ops[[same[0] + 1, same[0]]]
    assert shard.canonical_checksum(x) != base
    x = copy.deepcopy(cs)
    x.section_begin[1] -= 1
    assert shard.canonical_checksum(x) != base


# ------------------------------------------------------------------ the torch.distributed data path, 2 processes on gloo

def _launch(nproc, port, *worker_args, timeout=900):
    import json, os, subprocess, sys
    from pathlib import Path
    worker = Path(__file__).resolve().parent / "shard_worker.py"
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
                          "--master-port", str(port), str(worker), *[str(a) for a in worker_args]], capture_output=True, text=True, env=env, timeout=timeout)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])


def test_two_ranks_gloo_all_to_all():
    import __graft_entry__ as ge
    ge.build_hostsim()
    ge.build_oracle()
    d = _launch(2, 29541, "gloo", "randmodel", 21, 120)
    assert d["ok"] and d["world"] == 2 and d["n_ops"] > 50
    assert sum(d["homed"]) == 120 and min(d["homed"]) > 20
    assert min(d["sent"]) > 1000


def test_peer_exchange_host_logic_single_rank_gloo():
    """PeerExchange's host side (meta rows + arena handle + capacity in one all-gather, regrow agreement, barrier) with the
    hostsim engine: host arenas cannot be mapped across processes, so one rank — the multi-rank data path is the GPU tier's."""
    import __graft_entry__ as ge
    ge.build_hostsim()
    ge.build_oracle()
    d = _launch(1, 29545, "gloo", "randmodel", 22, 90, "peers")
    assert d["ok"] and d["world"] == 1 and d["n_ops"] > 30 and d["homed"] == [90]


def test_an_engine_error_on_one_rank_aborts_every_rank():
    """A contract violation only one rank can see must not leave the others waiting in the next collective."""
    import __graft_entry__ as ge
    ge.build_hostsim()
    d = _launch(2, 29543, "gloo", "randmodel", 2, 40, "badzone", timeout=300)
    assert len(d["raised"]) == 2 and all(d["raised"])
    assert any("zone table" in r for r in d["raised"])


@pytest.mark.gpu
def test_nccl_ranks_equal_unsharded():
    """One process per GPU, blobs over NCCL: needs >= 2 GPUs (skipped on a single-GPU machine)."""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least 2 GPUs")
    d = _launch(min(n, 8), 29547, "nccl", "synth", 4, 400_000)
    assert d["ok"] and d["n_ops"] > 100_000
    assert sum(d["homed"]) == d["n_objects"] and min(d["launches"]) > 0
    d = _launch(min(n, 8), 29549, "nccl", "synth", 4, 400_000, "peers")  # rows stored straight into the other GPUs' arenas (CUDA IPC)
    assert d["ok"] and d["n_ops"] > 100_000 and min(d["sent"]) > 0


# ------------------------------------------------------------------ GPU tier: several engines on one GPU, blobs in HBM

@pytest.mark.gpu
@pytest.mark.parametrize("seed,n_ranks", [(0, 2), (1, 3), (2, 4), (3, 8), (4, 1)])
def test_gpu_sharded_random_models(garecon, oracle, seed, n_ranks):
    objects, actual = randmodel.make(seed, n_objects=80)
    slices = shard.slice_model(objects, actual, n_ranks)
    engines, keep = [], []
    for objs_r, act_r, _ in slices:
        e = garecon.Engine(cluster_name="default")
        e.load(garecon.pack(objs_r, act_r))
        engines.append(e)
    shard.exchange_local(engines, [s[2] for s in slices], keep, device="cuda:0")
    parts = [e.diff() for e in engines]
    assert all(p.kernel_launches > 0 for p in parts)
    for e in engines:
        e.close()
    want = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    check_slices(garecon, want, parts, len(objects))


@pytest.mark.gpu
def test_gpu_sharded_hot_keys(garecon, oracle):
    objects, actual = hotkeys.make()
    slices = shard.slice_model(objects, actual, 4)
    engines, keep = [], []
    for objs_r, act_r, _ in slices:
        e = garecon.Engine(cluster_name="default")
        e.load(garecon.pack(objs_r, act_r))
        engines.append(e)
    shard.exchange_local(engines, [s[2] for s in slices], keep, device="cuda:0")
    parts = [e.diff() for e in engines]
    for e in engines:
        e.close()
    check_slices(garecon, oracle.diff(garecon.pack(objects, actual), "default", mode=1), parts, len(objects))


@pytest.mark.gpu
@pytest.mark.parametrize("peers", [False, True])
def test_gpu_sharded_long_strings(garecon, oracle, peers):
    objects, actual, want_update = long_string_model()
    slices = shard.slice_model(objects, actual, 3)
    engines, keep = [], []
    for objs_r, act_r, _ in slices:
        e = garecon.Engine(cluster_name="default")
        e.load(garecon.pack(objs_r, act_r))
        engines.append(e)
    if peers:
        shard.exchange_local_peers(engines, [s[2] for s in slices])
    else:
        shard.exchange_local(engines, [s[2] for s in slices], keep, device="cuda:0")
    parts = [e.diff() for e in engines]
    for e in engines:
        e.close()
    want = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    assert sorted(int(o["obj"]) for o in want.ops) == [k for k in range(14) if want_update[k]]
    check_slices(garecon, want, parts, len(objects))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,n_total,n_ranks", [(4, 400_000, 4), (5, 200_000, 8), (3, 200_000, 2)])
def test_gpu_sharded_equals_unsharded_at_scale(garecon, cfg, n_total, n_ranks):
    """The sharded result of a generator cluster equals the single-engine diff of the union, bit for bit (both on the GPU;
    the unsharded GPU path is itself pinned against the oracle at this size in test_gpu_large.py)."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    slices = synth.cluster_slices(cfg, n_total, n_ranks)
    union = garecon.tables.concat_slices(slices)
    with garecon.Engine(cluster_name="default") as e:
        e.load(union)
        want = e.diff()
    parts = run_sharded_slices(garecon, None, slices, device="cuda:0")
    check_slices(garecon, want, parts, n_total)
    assert len(want.ops) > n_total // 4
    parts = run_sharded_slices(garecon, None, slices, device="cuda:0", peers=True)  # the peer-memory exchange (same process: plain pointers)
    check_slices(garecon, want, parts, n_total)
