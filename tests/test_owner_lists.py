"""Owner-keyed joins resolved once from the AWS side: every owner value and owner-keyed accelerator carries the canonical row of
the object its key names, and every object reads the per-object owned lists (accelerators in ListAccelerators order, owner
values in row order) instead of probing an owner index.  ix_owner / ix_val are built only for the deleted keys of gar_diff_keys.

The models below stress what the lists must get right: a load that repeats an object key (every row with the key sees the
same accelerators and values), keys that are not 3-part (an object namespace holding a '/', owners with no '/' at all), an
owner with more values than one warp step (40) and more than the per-list ordering takes (60: the stable radix fallback),
guest accelerators of sharded mode, deleted keys before and after a full diff, and object and AWS deltas in between.  Every
answer is checked against the oracle; hostsim runs the device code on the CPU, the GPU tier runs the same scenarios."""
import copy
import importlib

import numpy as np
import pytest

import randmodel
from test_object_deltas import Mirror, assert_same_full, key_of

shard = importlib.import_module("aws-global-accelerator-controller_b200.shard")

NONE = 0xFFFFFFFF
ANN = randmodel.ANN
OWNER = "aws-global-accelerator-owner"


def owner_of(acc):
    return dict(acc["tags"]).get(OWNER, "")


def owner_value(owner):
    return f'"heritage=aws-global-accelerator-controller,cluster=default,{owner}"'


def resource(ob):
    return f"{ob['kind']}/{ob['ns']}/{ob['name']}"


def retag(acc, owner):
    a = copy.deepcopy(acc)
    a["tags"] = [(k, owner if k == OWNER else v) for k, v in a["tags"]]
    a["arn"] += "-" + owner.replace("/", "-")
    return a


def owner_model(seed, hot_values):
    """randmodel cluster plus: a duplicated key, a key with two '/', owners without a 3-part key, and one hot owner."""
    objects, actual = randmodel.make(seed, n_objects=30)
    accs, zones = actual["accelerators"], actual["zones"]
    ga_owned = [i for i, ob in enumerate(objects) if any(owner_of(a) == resource(ob) for a in accs)
                and ob["lb_ingress"] and ".elb." in ob["lb_ingress"][0]]
    r53_owned = [i for i, ob in enumerate(objects) if ANN + "route53-hostname" in ob["annotations"]]
    assert len(ga_owned) >= 3 and r53_owned
    # the same key at a later row (another lbIngress list) and at the end: both copies must see the first row's lists
    d = ga_owned[0]
    dup = copy.deepcopy(objects[d])
    dup["lb_ingress"] = list(reversed(dup["lb_ingress"])) or ["x.example.com"]
    objects = objects[:d + 5] + [dup] + objects[d + 5:] + [copy.deepcopy(objects[d])]
    # a key with two '/': namespace "team/a"; copies of another object's accelerators and owner records name it
    src = objects[ga_owned[1] + (1 if ga_owned[1] > d + 4 else 0)]
    two = copy.deepcopy(src)
    two["ns"] = "team/a"
    objects.append(two)
    for a in [a for a in accs if owner_of(a) == resource(src)]:
        accs.append(retag(a, resource(two)))
    for z in zones:
        z["records"] += [dict(r, values=[owner_value(resource(two)) for v in r["values"]]) for r in z["records"]
                         if r.get("values") and owner_value(resource(src)) in r["values"]]
    # owners whose key is not 3-part: no object can have it (no '/'), or no object has it (two '/', not in the cache)
    for owner in ("service/lonely", "ingress/team/b/gone"):
        accs.append(retag(accs[0], owner))
        zones[0]["records"].append({"name": f"odd-{len(owner)}.{zones[0]['name']}", "type": "TXT", "values": [owner_value(owner)]})
    # one owner with many values in one zone, half of them with an alias A record under the same name
    hot = objects[r53_owned[0]]
    zone = next(z for z in zones if z["name"] == "example.com.")
    for k in range(hot_values):
        rn = f"hot{k}.example.com."
        zone["records"].append({"name": rn, "type": "TXT", "values": [owner_value(resource(hot))]})
        if k % 2:
            zone["records"].append({"name": rn, "type": "A", "alias": "x.awsglobalaccelerator.com."})
    hot["annotations"][ANN + "route53-hostname"] = "hot3.example.com,hot4.example.com,hot7.example.com"
    return objects, actual


def check_full(garecon, oracle, e, objects, actual):
    got = e.diff()
    want = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    return got


def check_keys(garecon, oracle, e, objects, actual, rows, deleted):
    got = e.diff_keys(rows, deleted)
    want = oracle.diff_keys(garecon.pack(objects, actual), rows, deleted, mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    return got


def deleted_keys(objects):
    """keys that own accelerators and values, the duplicated key, a 2-'/' key that is not in the cache, an unknown key"""
    return [key_of(objects[-2]), key_of(objects[0]), (1, "team/b/gone"), (0, "default/never")]


def scenario_duplicates_and_odd_keys(garecon, oracle, e, hot_values):
    objects, actual = owner_model(11, hot_values)
    snap = garecon.pack(objects, actual)
    e.load(snap)
    keys = [key_of(ob) for ob in objects]
    dups = [i for i, k in enumerate(keys) if keys.count(k) > 1]
    assert len(dups) == 3
    # deleted keys before any full diff (ix_owner / ix_val built on demand), then the full diff, then again
    check_keys(garecon, oracle, e, objects, actual, dups + [len(objects) - 1], deleted_keys(objects))
    got = check_full(garecon, oracle, e, objects, actual)
    check_keys(garecon, oracle, e, objects, actual, list(range(len(objects))), deleted_keys(objects))
    check_full(garecon, oracle, e, objects, actual)
    # the copy at the end (same lbIngress list) acts on the same accelerators as the first row
    ga = got.ops[:int(got.section_begin[1])]
    acc_ops = [[(int(op["head"]), int(op["a0"])) for op in ga if op["obj"] == r] for r in (dups[0], dups[2])]
    assert acc_ops[0] and acc_ops[0] == acc_ops[1]
    return objects, actual, snap


def scenario_object_delta(garecon, oracle, e, hot_values):
    objects, actual, snap = scenario_duplicates_and_odd_keys(garecon, oracle, e, hot_values)
    m = Mirror(objects, snap)
    keys = [key_of(ob) for ob in objects]
    first_dup = next(i for i, k in enumerate(keys) if keys.count(k) > 1)
    upd = copy.deepcopy(objects[-1])
    upd["lb_ingress"] = list(objects[3]["lb_ingress"])
    # delete the lowest row of the duplicated key (a later copy becomes canonical) and update the 2-'/' object
    deleted = [keys[first_dup]]
    usnap = garecon.pack([upd], None)
    res = e.apply_objects(usnap.objects, deleted)
    up_row, del_row, moved, _ = m.apply([upd], deleted, usnap)
    assert (res.upsert_row.tolist(), res.deleted_row.tolist(), res.moved_from.tolist()) == (up_row, del_row, moved)
    msnap = garecon.pack(m.objects, actual)
    got = e.diff_keys(up_row + [0, len(m.objects) - 1], deleted_keys(m.objects))
    want = oracle.diff_keys(msnap, up_row + [0, len(m.objects) - 1], deleted_keys(m.objects), mode=1)
    assert got.diff(want) == [], got.describe_first_mismatch(want)
    assert_same_full(e.diff(), oracle.diff(msnap, "default", mode=1), m.slab, msnap.arrays["o.slab"])


def scenario_aws_delta(garecon, oracle, e, hot_values):
    objects, actual, _ = scenario_duplicates_and_odd_keys(garecon, oracle, e, hot_values)
    accs = actual["accelerators"]
    owned = [r for r, a in enumerate(accs) if owner_of(a) in (resource(objects[-2]), resource(objects[-1]))]
    assert owned
    extra = retag(accs[owned[0]], resource(objects[-1]))  # appended: the owner's list grows by a row at the end
    rows = garecon.pack([], {"accelerators": [extra]})
    e.apply_actual(rows.actual, acc_target=[NONE], acc_deleted=[owned[0]])
    after = dict(actual, accelerators=[a for r, a in enumerate(accs) if r != owned[0]] + [extra])
    check_full(garecon, oracle, e, objects, after)
    check_keys(garecon, oracle, e, objects, after, [len(objects) - 1, len(objects) - 2], deleted_keys(objects))


SCENARIOS = {"duplicates_and_odd_keys": scenario_duplicates_and_odd_keys, "object_delta": scenario_object_delta, "aws_delta": scenario_aws_delta}


@pytest.fixture(scope="module")
def hostsim(garecon):
    import __graft_entry__ as ge
    lib = garecon.abi.load_library(ge.build_hostsim())
    e = garecon.Engine(cluster_name="default", lib=lib)
    yield e
    e.close()


@pytest.mark.parametrize("hot_values", [40, 60])
@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
def test_hostsim_owner_lists(garecon, oracle, hostsim, scenario, hot_values):
    SCENARIOS[scenario](garecon, oracle, hostsim, hot_values)


def test_hostsim_owner_lists_tiny_capacities(garecon, oracle, hostsim, monkeypatch):
    monkeypatch.setenv("GAR_TINY_CAPS", "1")
    scenario_object_delta(garecon, oracle, hostsim, 40)


def sharded_equals_unsharded(garecon, oracle, n_ranks, device="cpu", **engine_kw):
    """Guest accelerators (copies that answer by-target-hostname lookups on another shard) are never resolved to an owner:
    the merged sharded change set equals the unsharded one."""
    objects, actual = owner_model(12, 40)
    engines, keep = [], []
    slices = shard.slice_model(objects, actual, n_ranks)
    for objs_r, act_r, _ in slices:
        e = garecon.Engine(cluster_name="default", **engine_kw)
        snap = garecon.pack(objs_r, act_r)
        e.load(snap)
        engines.append(e)
        keep.append(snap)
    shard.exchange_local(engines, [s[2] for s in slices], keep, device=device)
    parts = [e.diff() for e in engines]
    for e in engines:
        e.close()
    got = shard.merge_changesets(parts, len(objects))
    want = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    assert np.array_equal(got["status_ga"], want.status_ga) and np.array_equal(got["status_r53"], want.status_r53)
    assert got["ops"].tolist() == want.ops.tolist()


@pytest.mark.parametrize("n_ranks", [2, 3])
def test_hostsim_sharded_guest_accelerators(garecon, oracle, n_ranks):
    import __graft_entry__ as ge
    sharded_equals_unsharded(garecon, oracle, n_ranks, lib=garecon.abi.load_library(ge.build_hostsim()))


# ------------------------------------------------------------------ GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("hot_values", [40, 60])
@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
def test_gpu_owner_lists(garecon, oracle, scenario, hot_values):
    with garecon.Engine(cluster_name="default", device=0) as e:  # a fresh engine: the 60-value lists switch it to the radix build
        SCENARIOS[scenario](garecon, oracle, e, hot_values)


@pytest.mark.gpu
@pytest.mark.parametrize("n_ranks", [2, 3])
def test_gpu_sharded_guest_accelerators(garecon, oracle, n_ranks):
    sharded_equals_unsharded(garecon, oracle, n_ranks, device="cuda:0")
