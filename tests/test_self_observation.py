"""Self-observation (include/garecon.h): from the second lbIngress that reaches the update/create stage on — and for a
hostname repeated in the route53 annotation — an object's ops are what the reference decides AFTER its own earlier ops, as its
per-key loop re-lists AWS between iterations (global_accelerator.go:133-157, :987-1002; route53.go:92-124).

Pinned three ways: expectations derived by hand from the Go source; oracle/pyref.py, which SIMULATES the reference literally
(an object-local overlay of everything its ops changed, every list call re-evaluated on it) against the closed-form rules of
oracle/oracle.cpp; and the device code (hostsim here, the sm_90a library in the GPU tier) against the oracle."""
import importlib

import numpy as np
import pytest

import executor
import multilbi

pyref = importlib.import_module("oracle.pyref")
ANN = multilbi.ANN
N, P = 0xFFFFFFFF, 0xFFFFFFFE
OK, OK_CREATED, R53_CLEANED = 1, 1 | (1 << 16), 1 | (2 << 16)  # no route53 annotation: CleanupRecordSet ran (route53/service.go:54-69)
CREATE_CHAIN, UPDATE_ACCEL, CREATE_LISTENER, UPDATE_LISTENER, CREATE_EG, UPDATE_EG, DELETE_CHAIN, R53_CREATE, R53_UPSERT = 1, 2, 3, 4, 5, 6, 7, 8, 9


def nlb(i, region="us-east-1"):
    name = f"{i:032x}"
    host = f"{name}-{i:016x}.elb.{region}.amazonaws.com"
    return host, {"region": region, "name": name, "dns": host, "arn": f"arn:lb:{i}", "state": "active"}


def svc(name, hosts, **ann):
    a = {ANN + "global-accelerator-managed": "true", "service.beta.kubernetes.io/aws-load-balancer-type": "nlb"}
    a.update({ANN + k.replace("_", "-"): v for k, v in ann.items()})
    return dict(kind="service", ns="default", name=name, spec_type="LoadBalancer", annotations=a, ports=[(80, "TCP"), (443, "TCP")], lb_ingress=hosts)


def acc(i, owner, thost, endpoints, name=None, n_lis=1, n_eg=1, extra=()):
    tags = [("aws-global-accelerator-controller-managed", "true"), ("aws-global-accelerator-owner", owner),
            ("aws-global-accelerator-target-hostname", thost), ("aws-global-accelerator-cluster", "default")] + list(extra)
    lis = [{"arn": f"l{i}{x}", "proto": "TCP", "ports": [80, 443], "egs": [{"arn": f"e{i}{x}{y}", "endpoints": list(endpoints)} for y in range(n_eg)]} for x in range(n_lis)]
    return {"arn": f"a{i}", "name": name or "service-default-" + owner.split("/")[-1], "dns": f"a{i}.awsglobalaccelerator.com", "enabled": True, "tags": tags, "listeners": lis}


def ga_ops(cs):
    sb = [int(x) for x in cs.section_begin]
    return [(int(o["head"]) & 0xFF, int(o["sub"]), int(o["a0"]), int(o["a1"]), int(o["a2"])) for o in cs.ops[sb[0]:sb[1]]]


def r53_ops(cs):
    sb = [int(x) for x in cs.section_begin]
    return [(int(o["head"]) & 0xFF, int(o["sub"]), int(o["a0"]), int(o["a1"]), int(o["a2"])) for o in cs.ops[sb[2]:sb[3]]]


(h0, lb0), (h1, lb1), (h2, lb2) = nlb(1), nlb(2), nlb(3)
ZONE = {"id": "Z", "name": "example.com.", "records": []}
OV = '"heritage=aws-global-accelerator-controller,cluster=default,service/default/s"'

# name -> (objects, actual, expected GA ops (op, j, a0, a1, a2), expected R53 ops, (status_ga, status_r53) of object 0)
CASES = {
    # Go: j=0 list empty -> create (tags thost=h0, EG=[lb0]).  j=1: the list now holds it; acceleratorChanged: thost h0 != h1 -> update
    # (:291-296); listener found and equal; endpoint group found; endpointContainsLB(lb1) false -> updateEndpointGroup (:337-345).
    "create_then_update_pending": ([svc("s", [h0, h1])], {"lbs": [lb0, lb1]},
                                   [(CREATE_CHAIN, 0, 0, N, N), (UPDATE_ACCEL, 1, P, 1, N), (UPDATE_EG, 1, P, P, 1)], [], (OK_CREATED, R53_CLEANED)),
    # the same hostname twice: the second iteration finds everything in the state the first one left
    "same_hostname_twice": ([svc("s", [h0, h0])], {"lbs": [lb0]}, [(CREATE_CHAIN, 0, 0, N, N)], [], (OK_CREATED, R53_CLEANED)),
    # in sync with lb0: nothing at j=0; j=1 rewrites tag and endpoint group (the reference flip-flops such objects, one accelerator)
    "in_sync_then_rewrite": ([svc("s", [h0, h1])], {"lbs": [lb0, lb1], "accelerators": [acc(1, "service/default/s", h0, ["arn:lb:1"])]},
                             [(UPDATE_ACCEL, 1, 0, 1, N), (UPDATE_EG, 1, 0, 0, 1)], [], (OK, R53_CLEANED)),
    # endpoint group already lists both load balancers: only the tag moves
    "eg_holds_both": ([svc("s", [h0, h1])], {"lbs": [lb0, lb1], "accelerators": [acc(1, "service/default/s", h0, ["arn:lb:1", "arn:lb:2"])]},
                      [(UPDATE_ACCEL, 1, 0, 1, N)], [], (OK, R53_CLEANED)),
    # snapshot EG = [lb0, lb2]: j=1 replaces it by [lb1]; at j=2 it holds [lb1], NOT the snapshot's list -> replaced again
    "replaced_list_is_what_later_iterations_see": (
        [svc("s", [h0, h1, h2])], {"lbs": [lb0, lb1, lb2], "accelerators": [acc(1, "service/default/s", h0, ["arn:lb:1", "arn:lb:3"])]},
        [(UPDATE_ACCEL, 1, 0, 1, N), (UPDATE_EG, 1, 0, 0, 1), (UPDATE_ACCEL, 2, 0, 2, N), (UPDATE_EG, 2, 0, 0, 2)], [], (OK, R53_CLEANED)),
    # no listener: created at j=0 together with its endpoint group [lb0]; j=1 addresses that endpoint group as PENDING
    "listener_created_then_eg_pending": (
        [svc("s", [h0, h1])], {"lbs": [lb0, lb1], "accelerators": [acc(1, "service/default/s", h0, [], n_lis=0)]},
        [(CREATE_LISTENER, 0, 0, N, N), (CREATE_EG, 0, 0, N, 0), (UPDATE_ACCEL, 1, 0, 1, N), (UPDATE_EG, 1, 0, P, 1)], [], (OK, R53_CLEANED)),
    # a user tag overwrites the managed tag: what the object creates is never listed again -> the reference creates at every iteration
    "user_tag_hides_what_was_created": (
        [svc("s", [h0, h1], global_accelerator_tags="aws-global-accelerator-controller-managed=false")], {"lbs": [lb0, lb1]},
        [(CREATE_CHAIN, 0, 0, N, N), (CREATE_CHAIN, 1, 1, N, N)], [], (OK_CREATED, R53_CLEANED)),
    # a user tag pins target-hostname: acceleratorChanged no longer depends on the load balancer
    "user_tag_pins_target_hostname": (
        [svc("s", [h0, h1], global_accelerator_tags="aws-global-accelerator-target-hostname=x")], {"lbs": [lb0, lb1]},
        [(CREATE_CHAIN, 0, 0, N, N), (UPDATE_EG, 1, P, P, 1)], [], (OK_CREATED, R53_CLEANED)),
    # route53: a hostname repeated in the annotation is created once (route53.go:92-113: the second visit finds the record)
    "repeated_hostname_created_once": (
        [svc("s", [h0], route53_hostname="a.example.com,a.example.com,b.example.com")],
        {"lbs": [lb0], "accelerators": [acc(1, "service/default/s", h0, ["arn:lb:1"])], "zones": [ZONE]},
        [], [(R53_CREATE, 0, 0, 0, N), (R53_CREATE, 2, 0, 0, N)], (OK, OK_CREATED)),
    # route53 with two lbIngress served by different accelerators: the record created for accelerator 0 is re-pointed to accelerator 1
    "second_lbingress_repoints_pending_record": (
        [svc("s", [h0, h1], route53_hostname="a.example.com")],
        {"lbs": [lb0, lb1], "accelerators": [acc(1, "service/default/s", h0, ["arn:lb:1", "arn:lb:2"]), acc(2, "service/other/t", h1, [], name="x")], "zones": [ZONE]},
        [(UPDATE_ACCEL, 1, 0, 1, N)], [(R53_CREATE, 0, 0, 0, N), (R53_UPSERT, (1 << 20) | 0, 0, 1, P)], (OK, OK_CREATED)),
    # ... and an existing, in-sync record is re-pointed by row
    "second_lbingress_repoints_existing_record": (
        [svc("s", [h0, h1], route53_hostname="a.example.com")],
        {"lbs": [lb0, lb1], "accelerators": [acc(1, "service/default/s", h0, ["arn:lb:1", "arn:lb:2"]), acc(2, "service/other/t", h1, [], name="x")],
         "zones": [dict(ZONE, records=[{"name": "a.example.com.", "type": "TXT", "values": [OV]}, {"name": "a.example.com.", "type": "A", "alias": "a1.awsglobalaccelerator.com."}])]},
        [(UPDATE_ACCEL, 1, 0, 1, N)], [(R53_UPSERT, (1 << 20) | 0, 0, 1, 1)], (OK, OK)),
}


def _check_case(name, cs):
    objects, actual, want_ga, want_r53, (st_ga, st_r53) = CASES[name]
    assert ga_ops(cs) == want_ga, name
    assert r53_ops(cs) == want_r53, name
    assert int(cs.status_ga[0]) == st_ga and int(cs.status_r53[0]) == st_r53, name


@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_derived_expectations_pin_the_oracle(garecon, oracle, name):
    objects, actual = CASES[name][:2]
    snap = garecon.pack(objects, actual)
    _check_case(name, oracle.diff(snap, "default", mode=0))
    _check_case(name, oracle.diff(snap, "default", mode=1))
    ref = pyref.diff(objects, actual, "default")  # the literal simulation agrees
    assert [tuple(o) for o in ref["ops"]] == [tuple(int(x) for x in o) for o in oracle.diff(snap, "default", mode=1).ops.tolist()]


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    e = garecon.Engine(cluster_name="default", lib=garecon.abi.load_library(ge.build_hostsim()))
    yield e
    e.close()


@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_derived_expectations_on_the_device_logic(garecon, hostsim, name):
    snap = garecon.pack(*CASES[name][:2])  # hostsim reads the columns in place: keep the snapshot alive
    hostsim.load(snap)
    _check_case(name, hostsim.diff())


@pytest.mark.parametrize("seed", range(40))
def test_closed_form_rules_equal_the_literal_simulation(garecon, oracle, seed):
    objects, actual = multilbi.make(seed)
    snap = garecon.pack(objects, actual)
    want = oracle.diff(snap, "default", mode=1)
    assert oracle.diff(snap, "default", mode=0).diff(want) == []
    ref = pyref.diff(objects, actual, "default")
    assert [tuple(o) for o in ref["ops"]] == [tuple(int(x) for x in o) for o in want.ops.tolist()]
    assert ref["status_ga"] == want.status_ga.tolist() and ref["status_r53"] == want.status_r53.tolist()


@pytest.mark.parametrize("seed", range(40, 60))
def test_device_logic_equals_oracle_on_multi_lbingress_models(garecon, oracle, hostsim, seed):
    snap = garecon.pack(*multilbi.make(seed))
    hostsim.load(snap)
    got = hostsim.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


def _converge(garecon, diff_fn, objects, actual, rounds=5):
    sizes = []
    for _ in range(rounds):
        cs = diff_fn(garecon.pack(objects, actual))
        actual = executor.apply(objects, actual, cs)
        sizes.append(len(cs.ops))
    return actual, sizes


def test_two_lbingress_object_owns_exactly_one_accelerator(garecon, oracle):
    """ADVICE r1: a frozen-snapshot evaluation created one accelerator per lbIngress and never deleted the duplicate.  With
    self-observation the batch creates ONE and updates it, like the reference; later batches keep rewriting that one
    accelerator (the reference flip-flops too) but never add another."""
    objects = [svc("s", [h0, h1])]
    actual = {"lbs": [lb0, lb1], "accelerators": [], "zones": [dict(ZONE)]}
    final, sizes = _converge(garecon, lambda s: oracle.diff(s, "default", mode=1), objects, actual)
    mine = [a for a in final["accelerators"] if ("aws-global-accelerator-owner", "service/default/s") in [tuple(t) for t in a["tags"]]]
    assert len(mine) == 1 and len(final["accelerators"]) == 1
    assert len(mine[0]["listeners"]) == 1 and len(mine[0]["listeners"][0]["egs"]) == 1
    assert sizes[1:] == [sizes[1]] * (len(sizes) - 1)  # a periodic steady state: the same rewrite every batch, nothing new


def test_repeated_route53_hostname_gets_one_record_pair(garecon, oracle):
    """A hostname written twice in the annotation: one TXT + one A record after the first batch (a second R53_CREATE for the
    same name would be rejected by Route53), nothing left to do in the second."""
    objects = [svc("s", [h0], route53_hostname="a.example.com,a.example.com")]
    actual = {"lbs": [lb0], "accelerators": [acc(1, "service/default/s", h0, ["arn:lb:1"])], "zones": [dict(ZONE)]}
    final, sizes = _converge(garecon, lambda s: oracle.diff(s, "default", mode=1), objects, actual, rounds=3)
    assert sorted(r["type"] for r in final["zones"][0]["records"] if r["name"] == "a.example.com.") == ["A", "TXT"]
    assert sizes == [1, 0, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_gpu_hand_derived_expectations(garecon, engine, name):
    engine.load(garecon.pack(*CASES[name][:2]))
    _check_case(name, engine.diff())


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(60, 90))
def test_gpu_equals_oracle_on_multi_lbingress_models(garecon, oracle, engine, seed):
    snap = garecon.pack(*multilbi.make(seed, n_objects=60))
    engine.load(snap)
    got = engine.diff()
    want = oracle.diff(snap, "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)


@pytest.mark.gpu
def test_gpu_two_lbingress_object_owns_exactly_one_accelerator(garecon, engine):
    objects = [svc("s", [h0, h1]), svc("t", [h2], route53_hostname="a.example.com,a.example.com")]
    actual = {"lbs": [lb0, lb1, lb2], "accelerators": [acc(1, "service/default/t", h2, ["arn:lb:3"])], "zones": [dict(ZONE)]}

    def diff(snap):
        engine.load(snap)
        return engine.diff()
    final, _ = _converge(garecon, diff, objects, actual)
    assert len([a for a in final["accelerators"] if ("aws-global-accelerator-owner", "service/default/s") in [tuple(t) for t in a["tags"]]]) == 1
    assert sorted(r["type"] for r in final["zones"][0]["records"] if r["name"] == "a.example.com.") == ["A", "TXT"]
