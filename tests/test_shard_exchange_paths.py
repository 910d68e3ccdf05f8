"""Every data path of the sharded exchange, end to end, on poisoned buffers.

The in-process exchange helpers of shard.py zero their buffers, but DistExchange (one process per GPU) allocates its send and
receive buffers with torch.empty, and the peer arenas are plain allocations.  Here every send buffer, receive buffer (with the 64 bytes behind it) and peer arena
starts as POISON, and each set of engines runs one whole exchange before the one that is checked, so the engine-owned peer stage
holds stale non-zero bytes too.  Then:
  * every blob that travelled, per round and per (source, destination), is parsed with the layout of tests/shardblob.py and its
    live bytes (columns and every string's [off, off + len)) must equal those of every other path and of the host simulation;
  * the merged change set must equal the oracle (small models) or the unsharded GPU diff (generator clusters, which
    test_gpu_large.py pins against the oracle).

Paths: send buffer + all-to-all (default, GAR_PACK_TMA=1 bulk-store pack, GAR_SHARD_COPY_MERGE=1 merged slabs copied) and peer
arenas (staged + k_peer_push, GAR_PEER_CE=1 copy engines, GAR_PEER_DIRECT=1 pack kernels store into the arenas, and
GAR_PACK_TMA=1 with either).  The host-simulation tier runs the same poisoned loops on the CPU."""
import ctypes as C
import importlib

import numpy as np
import pytest

import hotkeys
import multilbi
import randmodel
import shardblob as sb
from test_sharded import check_slices, long_string_model

shard = importlib.import_module("aws-global-accelerator-controller_b200.shard")

POISON = 0xA5
SWITCHES = ("GAR_PACK_TMA", "GAR_SHARD_COPY_MERGE", "GAR_PEER_CE", "GAR_PEER_DIRECT")
VARIANTS = {
    "a2a": ("a2a", {}),
    "a2a_tma": ("a2a", {"GAR_PACK_TMA": "1"}),
    "a2a_copy_merge": ("a2a", {"GAR_SHARD_COPY_MERGE": "1"}),
    "peers": ("peers", {}),
    "peers_ce": ("peers", {"GAR_PEER_CE": "1"}),
    "peers_direct": ("peers", {"GAR_PEER_DIRECT": "1"}),
    "peers_tma": ("peers", {"GAR_PACK_TMA": "1"}),
    "peers_tma_direct": ("peers", {"GAR_PACK_TMA": "1", "GAR_PEER_DIRECT": "1"}),
}


# ------------------------------------------------------------------ buffers

class _DevBytes:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 3}


def _sync(device):
    if device != "cpu":
        import torch
        torch.cuda.synchronize()


def _poison_raw(ptr, nbytes, device):
    """Fill an engine-owned arena (device or host memory) with POISON."""
    if device == "cpu":
        C.memset(ptr, POISON, nbytes)
    else:
        import torch
        torch.as_tensor(_DevBytes(ptr, nbytes), device=device).fill_(POISON)
        torch.cuda.synchronize()


def _read_raw(ptr, nbytes, device):
    if device == "cpu":
        return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr)).copy()
    import torch
    return torch.as_tensor(_DevBytes(ptr, nbytes), device=device).cpu().numpy()


def _blob_offsets(meta, g):
    """all_meta[s][d] -> offset of each source's blob inside destination d's receive buffer"""
    return [np.concatenate([[0], np.cumsum([sb.blob_bytes(meta[s][d]) for s in range(g)])]).astype(np.int64) for d in range(g)]


# ------------------------------------------------------------------ exchange loops (every buffer poisoned)

def exchange_a2a(engines, shards, keep, device):
    """shard.exchange_local with torch.full(POISON) buffers.  -> per round (all_meta [s][d], {(s, d): blob bytes})"""
    import torch
    g, out = len(engines), []
    for rnd in (1, 2):
        metas, sends = [], []
        for e, sh in zip(engines, shards):
            meta, nbytes = e.shard_route(sh, rnd)
            assert [e.blob_bytes(meta[d]) for d in range(g)] == [int(x) for x in nbytes] == [sb.blob_bytes(meta[d]) for d in range(g)]
            buf = torch.full((int(nbytes.sum()) + 64,), POISON, dtype=torch.uint8, device=device)
            _sync(device)
            e.shard_pack(buf.data_ptr())
            keep.append(buf)
            metas.append(meta)
            sends.append((buf, np.concatenate([[0], np.cumsum(nbytes)]).astype(np.int64)))
        blobs = {(s, d): sends[s][0][int(sends[s][1][d]):int(sends[s][1][d + 1])].cpu().numpy() for s in range(g) for d in range(g)}
        for d, e in enumerate(engines):
            recv_meta = np.stack([metas[s][d] for s in range(g)])
            n = int(sum(len(blobs[s, d]) for s in range(g)))
            recv = torch.full((n + 64,), POISON, dtype=torch.uint8, device=device)
            p = 0
            for s in range(g):
                part = sends[s][0][int(sends[s][1][d]):int(sends[s][1][d + 1])]
                recv[p:p + len(part)] = part
                p += len(part)
            _sync(device)
            keep.append(recv)
            e.shard_unpack(rnd, recv.data_ptr(), recv_meta)
        out.append((np.stack(metas), blobs))
    return out


def exchange_peers(engines, shards, device):
    """shard.exchange_local_peers with every arena poisoned over its whole capacity before the packs."""
    g, out = len(engines), []
    for rnd in (1, 2):
        all_meta = np.stack([e.shard_route(sh, rnd)[0] for e, sh in zip(engines, shards)])
        arenas, handles = [], []
        for d, e in enumerate(engines):
            need = sum(e.blob_bytes(all_meta[s][d]) for s in range(g))
            ptr, h, cap = e.shard_arena(rnd, need)
            assert cap >= need + 64
            _poison_raw(ptr, cap, device)
            arenas.append((ptr, need))
            handles.append(h)
        for e in engines:
            e.shard_open_peers(rnd, np.stack(handles))
        for e in engines:
            e.shard_pack_peers(rnd, all_meta)
        offs = _blob_offsets(all_meta, g)
        blobs = {}
        for d in range(g):
            raw = _read_raw(arenas[d][0], arenas[d][1] + 64, device)
            assert (raw[arenas[d][1]:] == POISON).all(), f"round {rnd}: bytes behind destination {d}'s blobs were written"
            for s in range(g):
                blobs[s, d] = raw[offs[d][s]:offs[d][s + 1]]
        for d, e in enumerate(engines):
            e.shard_unpack(rnd, arenas[d][0], np.ascontiguousarray(all_meta[:, d]))
        out.append((all_meta, blobs))
    return out


def run_path(garecon, lib, snaps, shards, kind, device):
    """Load the slices, run one poisoned exchange and diff, then the checked one on the same engines.
    -> (parts of the first exchange, parts of the second, blobs of the second)"""
    engines, keep = [], []
    for snap in snaps:
        e = garecon.Engine(cluster_name="default", lib=lib)
        e.load(snap)
        engines.append(e)
    try:
        results = []
        for _ in range(2):
            rounds = exchange_a2a(engines, shards, keep, device) if kind == "a2a" else exchange_peers(engines, shards, device)
            results.append(([e.diff() for e in engines], rounds))
        return results[0][0], results[1][0], results[1][1]
    finally:
        for e in engines:
            e.close()


def live(rounds):
    """per round: meta rows and the live bytes of every (source, destination) blob"""
    return [(meta, {k: sb.live_bytes(b, meta[k[0]][k[1]]) for k, b in blobs.items()}) for meta, blobs in rounds]


def assert_same_blobs(ref, got, what):
    for rnd, ((m0, b0), (m1, b1)) in enumerate(zip(ref, got), 1):
        assert np.array_equal(m0, m1), f"{what}: round {rnd} meta rows differ"
        for k in b0:
            if not np.array_equal(b0[k], b1[k]):
                bad = np.flatnonzero(b0[k] != b1[k]) if len(b0[k]) == len(b1[k]) else [-1]
                raise AssertionError(f"{what}: round {rnd} blob {k[0]} -> {k[1]}: live bytes differ (first at live byte {int(bad[0])} of {len(b0[k])})")


def _clear(monkeypatch, env):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# ------------------------------------------------------------------ models

def dict_model(name):
    if name.startswith("rand"):
        return randmodel.make(int(name[4:]), n_objects=80)
    if name == "multilbi":
        return multilbi.make(3, n_objects=60)
    if name == "hotkeys":
        return hotkeys.make()
    return long_string_model()[:2]


def sliced(garecon, objects, actual, n_ranks):
    sl = shard.slice_model(objects, actual, n_ranks)
    return [garecon.pack(o, a) for o, a, _ in sl], [s for _, _, s in sl]


def check_oracle(garecon, oracle, objects, actual, parts):
    check_slices(garecon, oracle.diff(garecon.pack(objects, actual), "default", mode=1), parts, len(objects))


@pytest.fixture(scope="module")
def hostlib(garecon):
    import __graft_entry__ as ge
    return garecon.abi.load_library(ge.build_hostsim())


# ------------------------------------------------------------------ host simulation tier

@pytest.mark.parametrize("model,n_ranks", [("rand0", 2), ("rand1", 3), ("long", 3), ("long", 2)])
@pytest.mark.parametrize("kind", ["a2a", "peers"])
@pytest.mark.parametrize("copy_merge", [False, True], ids=["in_place", "copy_merge"])
def test_hostsim_poisoned_exchange(garecon, oracle, hostlib, monkeypatch, model, n_ranks, kind, copy_merge):
    """The device code compiled for the host, on poisoned buffers: results equal the oracle whether the merged sub-snapshot
    reads its strings from the receive buffers or from copied slabs, and both paths carry the same live bytes."""
    _clear(monkeypatch, {"GAR_SHARD_COPY_MERGE": "1"} if copy_merge else {})
    objects, actual = dict_model(model)
    snaps, shards = sliced(garecon, objects, actual, n_ranks)
    first, second, rounds = run_path(garecon, hostlib, snaps, shards, kind, "cpu")
    check_oracle(garecon, oracle, objects, actual, first)
    check_oracle(garecon, oracle, objects, actual, second)
    live(rounds)  # every blob parses: offsets follow the lengths, strings fill the announced slab bytes


# ------------------------------------------------------------------ GPU tier

def gpu_variants(garecon, monkeypatch, snaps, shards, check, ref=None):
    """Every variant on the same slices: results checked, live blob bytes equal to `ref` (or to the first variant's)."""
    for name, (kind, env) in VARIANTS.items():
        with monkeypatch.context() as mp:
            _clear(mp, env)
            first, second, rounds = run_path(garecon, None, snaps, shards, kind, "cuda:0")
        check(first)
        check(second)
        got = live(rounds)
        if ref is None:
            ref = got
        else:
            assert_same_blobs(ref, got, name)
    return ref


@pytest.mark.gpu
@pytest.mark.parametrize("n_ranks", [2, 3, 8])
@pytest.mark.parametrize("model", ["rand0", "rand1", "multilbi", "hotkeys", "long"])
def test_gpu_exchange_paths_small_models(garecon, oracle, hostlib, monkeypatch, model, n_ranks):
    objects, actual = dict_model(model)
    snaps, shards = sliced(garecon, objects, actual, n_ranks)
    _clear(monkeypatch, {})
    _, _, host_rounds = run_path(garecon, hostlib, snaps, shards, "a2a", "cpu")
    gpu_variants(garecon, monkeypatch, snaps, shards, lambda parts: check_oracle(garecon, oracle, objects, actual, parts), ref=live(host_rounds))


N_GEN = 199_992  # 2*10^5 generator objects, a multiple of both rank counts (one generator chunk per rank)


@pytest.mark.gpu
@pytest.mark.parametrize("n_ranks", [3, 8])
def test_gpu_exchange_paths_generator_cluster(garecon, monkeypatch, n_ranks):
    """2*10^5 generator objects: every rank sends the others more than one 48 MiB push group of the staged peer path."""
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    slices = synth.cluster_slices(4, N_GEN, n_ranks)
    union = garecon.tables.concat_slices(slices)
    with garecon.Engine(cluster_name="default") as e:
        e.load(union)
        want = e.diff()
    assert len(want.ops) > 50_000
    snaps = [garecon.tables.from_columns(o, a) for o, a in slices]
    ref = gpu_variants(garecon, monkeypatch, snaps, garecon.tables.shard_bases(slices), lambda parts: check_slices(garecon, want, parts, N_GEN))
    # what each rank sends the others in round 1: more than one of the staged peer path's 48 MiB push groups (105 MiB at 3
    # ranks, 52 MiB at 8)
    meta1 = ref[0][0]
    assert min(sum(sb.blob_bytes(meta1[s][d]) for d in range(n_ranks) if d != s) for s in range(n_ranks)) > 48 << 20


ANN = "aws-global-accelerator-controller.h3poteto.dev/"
TAG_M, TAG_O, TAG_H, TAG_C = ("aws-global-accelerator-controller-managed", "aws-global-accelerator-owner", "aws-global-accelerator-target-hostname",
                              "aws-global-accelerator-cluster")


def long_strings_at_scale(n=40_000, seed=5):
    """long_string_model at 4*10^4 Services: each one's global-accelerator-tags value equals a tag of its accelerator, except that
    on every third object the tag's LAST byte differs (that object needs GA_UPDATE_ACCEL).  Value lengths: mostly 2040-2057
    bytes (around the pack's 2 KB cut), every 50th 2-40 KB, one over 40 KB."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(2040 - 2, 2058 - 2, n)  # the annotation value is "k=" + value
    lens[::50] = rng.integers(2048, 40_000, len(lens[::50]))
    lens[n // 2 + 7] = 50_000
    alphabet = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789", dtype=np.uint8)
    pool = alphabet[rng.integers(0, len(alphabet), 60_000)].tobytes().decode()
    objects, lbs, accs, want_update = [], [], [], []
    for k in range(n):
        lbname = f"{k:032x}"
        host = f"{lbname}-0123456789abcdef.elb.us-west-2.amazonaws.com"
        at = (k * 7919) % 5000
        v = pool[at:at + int(lens[k])]
        off = k % 3 == 1
        want_update.append(off)
        objects.append(dict(kind="service", ns="default", name=f"s{k}", spec_type="LoadBalancer", ports=[(80, "TCP")], lb_ingress=[host],
                            annotations={ANN + "global-accelerator-managed": "true", "service.beta.kubernetes.io/aws-load-balancer-type": "nlb",
                                         ANN + "global-accelerator-tags": "k=" + v}))
        lbs.append({"region": "us-west-2", "name": lbname, "dns": host, "arn": f"arn:lb{k}", "state": "active"})
        accs.append({"arn": f"a{k}", "name": f"service-default-s{k}", "dns": f"a{k}.awsglobalaccelerator.com", "enabled": True,
                     "tags": [(TAG_M, "true"), (TAG_O, f"service/default/s{k}"), (TAG_H, host), (TAG_C, "default"), ("k", v[:-1] + "!" if off else v)],
                     "listeners": [{"arn": f"l{k}", "proto": "TCP", "ports": [80], "egs": [{"arn": f"e{k}", "endpoints": [f"arn:lb{k}"]}]}]})
    return objects, {"lbs": lbs, "accelerators": accs, "zones": []}, want_update


@pytest.mark.gpu
def test_gpu_exchange_paths_long_strings_at_scale(garecon, monkeypatch):
    """Enough selected rows with strings over 2 KB in the annotation and tag levels that FShPackLong's workers take a second
    stride; every byte of every long value must arrive, on every path."""
    objects, actual, want_update = long_strings_at_scale()
    with garecon.Engine(cluster_name="default") as e:
        e.load(garecon.pack(objects, actual))
        want = e.diff()
    sbeg = [int(x) for x in want.section_begin]
    ga = want.ops[sbeg[0]:sbeg[1]]
    assert [int(o["obj"]) for o in ga] == [k for k, u in enumerate(want_update) if u]
    assert all(int(o["head"]) & 0xFF == 2 for o in ga)  # GA_UPDATE_ACCEL
    snaps, shards = sliced(garecon, objects, actual, 2)
    ref = gpu_variants(garecon, monkeypatch, snaps, shards, lambda parts: check_slices(garecon, want, parts, len(objects)))
    # the pack's long-string pass had a second stride to take: some blob's annotation / tag level selected that many rows
    meta1, stride = ref[0][0], 132 * 8 * 256 // 8
    for s in range(2):
        assert sum(int(meta1[s][d][sb.L_ANN]) for d in range(2)) > stride and sum(int(meta1[s][d][sb.L_TAG]) for d in range(2)) > stride
