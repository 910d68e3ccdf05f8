"""CPU tier: the device row logic + pipeline (csrc/gar_rows.h, gar_pipeline.h) compiled for the host
(tests/hostsim, a test build) must produce the oracle's change set bit for bit.  The same comparison runs
against the real sm_90a library in test_gpu_parity.py."""
import ctypes as C

import pytest

import randmodel


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    path = ge.build_hostsim()
    lib = garecon.abi.load_library(path)
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


@pytest.mark.parametrize("seed", range(60))
def test_hostsim_matches_oracle(garecon, oracle, hostsim, seed):
    objects, actual = randmodel.make(seed, n_objects=40)
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    got = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


def test_hostsim_empty_snapshot(garecon, oracle, hostsim):
    snap = garecon.pack([], {})
    hostsim.load(snap)
    got = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == []
    assert len(got.ops) == 0


def test_hostsim_empty_cache_guard_and_no_orphans_flag(garecon, oracle):
    """include/garecon.h "Orphan sweep precondition" on the CPU tier (same pipeline text as the CUDA engine)."""
    import numpy as np
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    objects, actual = randmodel.make(12, n_objects=80)
    only_actual = garecon.pack([], actual)
    with garecon.Engine(cluster_name="default", lib=lib) as e:
        e.load(only_actual)
        with pytest.raises(garecon.abi.GarError, match="object table is empty"):
            e.diff()
    with garecon.Engine(cluster_name="default", lib=lib, allow_empty_cache=True) as e:
        e.load(only_actual)
        assert e.diff().diff(oracle.diff(only_actual, "default", mode=1)) == []
    snap = garecon.pack(objects[:40], actual)
    want = oracle.diff(snap, "default", mode=1)
    sb = [int(x) for x in want.section_begin]
    with garecon.Engine(cluster_name="default", lib=lib, orphans=False) as e:
        e.load(snap)
        got = e.diff()
    gb = [int(x) for x in got.section_begin]
    assert gb[2] == gb[1] and gb[4] == gb[3] and sb[2] > sb[1] and sb[4] > sb[3]
    assert np.array_equal(got.ops[gb[0]:gb[1]], want.ops[sb[0]:sb[1]]) and np.array_equal(got.ops[gb[2]:gb[3]], want.ops[sb[2]:sb[3]])


def test_hostsim_other_cluster_name(garecon, oracle):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    objects, actual = randmodel.make(3, n_objects=40, cluster="prod-1")
    snap = garecon.pack(objects, actual)
    with garecon.Engine(cluster_name="prod-1", lib=lib) as e:
        e.load(snap)
        got = e.diff()
    want = oracle.diff(snap, "prod-1", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert len(got.ops) > 10


def test_hostsim_hot_keys_force_the_fallback_paths(garecon, oracle, hostsim):
    import hotkeys
    objects, actual = hotkeys.make()
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    got = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    faithful = oracle.diff(snap, "default", mode=0)
    assert want.diff(faithful) == []
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert len(got.ops) > 200


def test_warp_emulation_catches_a_non_uniform_vote(garecon):
    """The hostsim warp emulator must flag a GAR_ANY that not every lane reaches (it would hang a real GPU)."""
    import ctypes, subprocess, tempfile, textwrap
    from pathlib import Path
    repo = Path(__file__).resolve().parent.parent
    src = textwrap.dedent(r'''
        #define main hostsim_unused_main
        #include "tests/hostsim/hostsim.cpp"
        #undef main
        struct Bad { GAR_HD void operator()(u32 i, bool valid) const { if (i % 2 == 0) (void)GAR_ANY(true); } };
        struct Good { GAR_HD void operator()(u32 i, bool valid) const { for (u32 k = 0; GAR_ANY(k < i % 5); k++) {} } };
        extern "C" int probe(int which) {
          gar_engine e;
          g_nonuniform_vote = false;
          if (which) e.for_each_warp("bad", 64, Bad{}); else e.for_each_warp("good", 64, Good{});
          return g_nonuniform_vote ? 1 : 0;
        }
    ''')
    with tempfile.TemporaryDirectory() as d:
        (Path(d) / "t.cpp").write_text(src)
        subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", str(repo), "-o", f"{d}/t.so", f"{d}/t.cpp"], check=True)
        lib = ctypes.CDLL(f"{d}/t.so")
        assert lib.probe(0) == 0
        assert lib.probe(1) == 1


def test_hostsim_tokeniser_fuzz(garecon, oracle, hostsim):
    import fuzzcases
    snap = garecon.pack(fuzzcases.fuzz_hostnames(11, 1500), {})
    hostsim.load(snap)
    got = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert len(set(got.tok_code.tolist())) >= 8


def test_hostsim_listen_ports_fuzz(garecon, oracle, hostsim):
    import fuzzcases
    snap = garecon.pack(fuzzcases.listen_objects(), {})
    hostsim.load(snap)
    got = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert len(got.dports) > 10


def test_hostsim_port_multisets(garecon, oracle, hostsim):
    """listenerPortChanged semantics (global_accelerator.go:458-492) on many list shapes: duplicates, permutations,
    prefixes, long lists — the kernel strips common prefix/suffix, the oracle builds the reference's count map."""
    import random
    rng = random.Random(3)
    ANN = "aws-global-accelerator-controller.h3poteto.dev/"
    host = "{:032x}-{:016x}.elb.us-east-1.amazonaws.com"
    objects, lbs, accs = [], [], []
    for i in range(300):
        n = rng.choice([0, 1, 2, 3, 5, 17, 64])
        want = [rng.choice([80, 443, 8080, 8443, 9000 + rng.randrange(50)]) for _ in range(n)]
        shape = rng.randrange(7)
        have = list(want)
        if shape == 1 and have:
            have[rng.randrange(len(have))] = 7
        elif shape == 2:
            have = have + [rng.choice(have) if have and rng.random() < 0.5 else 7]
        elif shape == 3 and have:
            have = have[:-1]
        elif shape == 4:
            rng.shuffle(have)
        elif shape == 5 and have:
            have = have + have
        elif shape == 6:
            have = [p for p in have if rng.random() < 0.7]
        h = host.format(i, i)
        name = f"svc{i}"
        objects.append(dict(kind="service", ns="d", name=name, annotations={ANN + "global-accelerator-managed": "true", "service.beta.kubernetes.io/aws-load-balancer-type": "nlb"},
                            lb_ingress=[h], ports=[(p, "TCP") for p in want]))
        arn = f"arn:lb:{i}"
        lbs.append(dict(region="us-east-1", name=f"{i:032x}", dns=h, arn=arn, state="active"))
        tags = [("aws-global-accelerator-controller-managed", "true"), ("aws-global-accelerator-owner", f"service/d/{name}"),
                ("aws-global-accelerator-target-hostname", h), ("aws-global-accelerator-cluster", "default")]
        accs.append(dict(arn=f"a{i}", name=f"service-d-{name}", dns="x", enabled=True, tags=tags,
                         listeners=[dict(arn="l", proto="TCP", ports=have, egs=[dict(arn="e", endpoints=[arn])])]))
    snap = garecon.pack(objects, dict(lbs=lbs, accelerators=accs))
    hostsim.load(snap)
    got = hostsim.diff()
    want_cs = oracle.diff(snap, "default", mode=0)
    assert got.diff(want_cs) == [], got.describe_first_mismatch(want_cs)
    assert 30 < len(got.ops) < 300


def test_hostsim_huge_value_lists(garecon, oracle, hostsim):
    """A TXT record set with > 4096 values takes the grid-wide branch of the record pass (FClassifyBigRecords); one with > 32
    values the block-wide one."""
    import hotkeys
    objects, actual = hotkeys.make(ndup_acc=3, ndup_alias=2, ndup_val=2100)
    assert max(len(r.get("values", [])) for r in actual["zones"][0]["records"]) > 4096
    snap = garecon.pack(objects, actual)
    hostsim.load(snap)
    got = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


@pytest.mark.parametrize("layout", ["level", "reverse", "shuffle"])
@pytest.mark.parametrize("seed", range(6))
def test_results_do_not_depend_on_the_slab_layout(garecon, oracle, hostsim, seed, layout):
    """Where the strings sit in the slabs is the packer's business: row-major by parent (the default), column-major, reversed
    or shuffled must give the same statuses and ops (string-ref outputs differ by construction)."""
    objects, actual = randmodel.make(seed, n_objects=40)
    base = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    snap = garecon.pack(objects, actual, layout=layout, seed=seed)
    hostsim.load(snap)
    got = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    for k in ("status_ga", "status_r53", "derived", "ops", "section_begin", "tok_code", "dport_begin", "dports"):
        assert getattr(got, k).tolist() == getattr(base, k).tolist(), k


def test_hostsim_capacity_overflow_paths(garecon, oracle, monkeypatch):
    """Intermediate relations whose size only the device knows (parsed ports, (object, hostname) pairs, ops) live in buffers
    with a capacity; a diff that outgrows one is re-run with a larger buffer.  GAR_TINY_CAPS=1 starts every capacity at 1, so
    every model takes those paths; the result must not change."""
    import __graft_entry__ as ge
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    lib = garecon.abi.load_library(ge.build_hostsim())
    for seed in range(8):
        objects, actual = randmodel.make(seed, n_objects=40)
        snap = garecon.pack(objects, actual)
        with garecon.Engine(cluster_name="default", lib=lib) as e:
            e.load(snap)
            got = e.diff()
            again = e.diff()
            keys = e.diff_keys(list(range(0, len(objects), 3)), [(0, "default/gone")])
        want = oracle.diff(snap, "default", mode=1)
        assert got.diff(want) == [], got.describe_first_mismatch(want)
        assert again.diff(want) == []
        wk = oracle.diff_keys(snap, list(range(0, len(objects), 3)), [(0, "default/gone")], cluster="default", mode=1)
        assert keys.diff(wk) == [], keys.describe_first_mismatch(wk)
