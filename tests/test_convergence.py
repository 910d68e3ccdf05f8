"""diff -> execute against a mock AWS model -> diff ... reaches a fixed point.

A size-independent property of the whole path (SURVEY.md §8 row f2): once the change set has been executed, the next
diff of every single-lbIngress object must be empty (statuses that are waiting states may persist).  Objects with
several lbIngress hostnames flip-flop in the reference too (each lbIngress rewrites the same accelerator,
global_accelerator.go:150-156), so they are excluded from the fixed-point assertion, not from parity.

The CPU tier runs it with the oracle and the warp-emulating hostsim build; the GPU tier with the sm_90a library."""
import copy

import numpy as np
import pytest

import executor
import randmodel


def _multi_lbi_rows(objects):
    """Objects that do not converge in the reference either: several lbIngress hostnames (each rewrites the same
    accelerator), or a tags annotation that overrides a system tag key (the accelerator it creates carries
    owner=<user value> last, so list-by-owner never finds it again: tagsContainsAllValues, later duplicate wins)."""
    out = set()
    claims = {}
    for i, ob in enumerate(objects):
        ann = dict(ob.get("annotations", {}))
        tags = ann.get("aws-global-accelerator-controller.h3poteto.dev/global-accelerator-tags", "")
        if len(ob.get("lb_ingress", [])) > 1 or "aws-global-accelerator-" in tags:
            out.add(i)
        for hn in ann.get("aws-global-accelerator-controller.h3poteto.dev/route53-hostname", "\0").split(","):
            claims.setdefault(hn, []).append(i)
    for hn, rows in claims.items():  # two owners of one hostname keep upserting the same alias record
        if hn != "\0" and len(rows) > 1:
            out.update(rows)
    return out


def _rounds(garecon, objects, actual, diff_fn, check_fn=None, max_rounds=6):
    history = []
    for _ in range(max_rounds):
        snap = garecon.pack(objects, actual)
        cs = diff_fn(snap)
        if check_fn:
            check_fn(snap, cs)
        history.append(cs)
        multi = _multi_lbi_rows(objects)
        live = [op for op in cs.ops.tolist() if not (op[1] != 0xFFFFFFFF and op[1] in multi)]
        if not live:
            return history
        actual = executor.apply(objects, actual, cs)
    raise AssertionError(f"no fixed point after {max_rounds} rounds; last round still has {len(live)} ops, e.g. {live[:3]}")


@pytest.mark.parametrize("seed", range(12))
def test_oracle_reaches_fixed_point(garecon, oracle, seed):
    objects, actual = randmodel.make(seed, n_objects=40)
    hist = _rounds(garecon, objects, actual, lambda s: oracle.diff(s, "default", mode=1))
    assert len(hist) >= 2 and len(hist[0].ops) > len(hist[-1].ops)


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


@pytest.mark.parametrize("seed", range(100, 106))
def test_device_logic_tracks_oracle_through_the_rounds(garecon, oracle, hostsim, seed):
    objects, actual = randmodel.make(seed, n_objects=40)

    def diff(snap):
        hostsim.load(snap)
        return hostsim.diff()

    def check(snap, cs):
        want = oracle.diff(snap, "default", mode=0)
        assert cs.diff(want) == [], cs.describe_first_mismatch(want)

    _rounds(garecon, objects, actual, diff, check)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(200, 212))
def test_gpu_tracks_oracle_through_the_rounds(garecon, oracle, engine, seed):
    objects, actual = randmodel.make(seed, n_objects=80)

    def diff(snap):
        engine.load(snap)
        return engine.diff()

    def check(snap, cs):
        want = oracle.diff(snap, "default", mode=1)
        assert cs.diff(want) == [], cs.describe_first_mismatch(want)

    hist = _rounds(garecon, objects, actual, diff, check)
    assert len(hist) >= 2
