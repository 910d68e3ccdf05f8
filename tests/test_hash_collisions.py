"""Keys that collide in tag and bucket at every hash-index probe of the engine.

An index entry keeps only the upper half of the 64-bit key hash (the tag), and the bucket is the low log2(nb) bits of the same
hash; every probe must follow a tag hit with a full key compare.  Random snapshots practically never contain two different keys
that agree on both (about r * m * 2**-32 per index), so these scenarios build them with collisions.find_pairs: in each one a
colliding impostor sits at a LOWER row (or earlier in list order) than the true match, so a probe that trusted the tag would
return the impostor.  Every scenario first asserts its preconditions (the index's bucket count under the engine's sizing rule is
within the bits the pair collides in, and the pair shares tag and bucket), then checks gar_diff, gar_diff_keys and, where they
apply, gar_bindings_diff and object deltas against the oracle, which keys its maps by the full strings.

The host simulation (tests/hostsim: the device row logic compiled for the CPU) runs every scenario; the GPU tier runs the same."""
import copy
import subprocess
import textwrap
from pathlib import Path

import numpy as np
import pytest

import collisions as C
from test_object_deltas import Mirror, assert_same_full, key_of

REPO = Path(__file__).resolve().parent.parent
CSRC = REPO / "aws-global-accelerator-controller_b200" / "csrc"
ANN = "aws-global-accelerator-controller.h3poteto.dev/"
REGION = "us-east-1"
BITS = 8  # every scenario keeps its tables within 2**8 buckets (each one asserts it)

# free-byte placements (collisions.OBJECT_KEYS has the object keys); each template is checked by collisions.placement_word
LB_NAMES = {"first": "{}-nlb-name", "middle": "nlbname-{}-x", "tail": "nlb-name-collide-{}"}
THOSTS = {"first": "{}ab-0123456789abcdef.elb.us-east-1.amazonaws.com", "middle": "web-nlb-{}-0123456789abcdef.elb.us-east-1.amazonaws.com"}
ZONE_NAMES = {"first": "{}.example.com", "middle": "zone-ab.{}.example.com", "tail": "zone-collide.com{}"}
RECORD_NAMES = {"first": "{}ab.example.com.", "middle": "records-{}.example.com."}
EG_ARN = "arn:aws:globalaccelerator::1:accelerator/a/listener/l/endpoint-group/eee{}"


def pair(fn, template, placement, seed=0, bits=BITS, fn_b=None):
    """one colliding pair whose keys differ only in the word `placement` names"""
    word = C.placement_word(template, placement)
    a, b = C.find_pairs(fn, template, 1, bits=bits, seed=seed, hash_fn_b=fn_b)[0]
    assert a != b and len(a) == len(b) and C.differing_words(a, b) == {word}
    return a, b


# ------------------------------------------------------------------ model builders (the dict model of tables.pack)

def lb_host(name):
    return f"{name}-0123456789abcdef.elb.{REGION}.amazonaws.com"


def lb(name, i, state="active"):
    return dict(region=REGION, name=name, dns=lb_host(name), arn=f"arn:aws:elasticloadbalancing:{REGION}:1:loadbalancer/net/{name}/{i:016x}", state=state)


def obj(kind, key, host, r53=None):
    ns, name = key.split("/", 1)
    ann = {ANN + "global-accelerator-managed": "true"}
    if r53:
        ann[ANN + "route53-hostname"] = r53
    if kind == "service":
        ann["service.beta.kubernetes.io/aws-load-balancer-type"] = "nlb"
        return dict(kind=kind, ns=ns, name=name, spec_type="LoadBalancer", annotations=ann, lb_ingress=[host], ports=[(80, "TCP")])
    return dict(kind=kind, ns=ns, name=name, ingress_class="alb", annotations=ann, lb_ingress=[host], ports=[80])


def accel(i, owner, thost, lb_arn=None, name="stale"):
    tags = [("aws-global-accelerator-controller-managed", "true"), ("aws-global-accelerator-owner", owner),
            ("aws-global-accelerator-target-hostname", thost), ("aws-global-accelerator-cluster", "default")]
    egs = [dict(arn=f"arn:aws:globalaccelerator::1:accelerator/c{i}/listener/0/endpoint-group/0", endpoints=[lb_arn] if lb_arn else [])]
    return dict(arn=f"arn:aws:globalaccelerator::1:accelerator/c{i}", name=name, dns=f"c{i:04d}.awsglobalaccelerator.com", enabled=True, tags=tags,
                listeners=[dict(arn=f"arn:aws:globalaccelerator::1:accelerator/c{i}/listener/0", proto="TCP", ports=[80], egs=egs)])


def owner_value(resource):
    return f'"heritage=aws-global-accelerator-controller,cluster=default,{resource}"'


def resource(ob):
    return f"{ob['kind']}/{ob['ns']}/{ob['name']}"


def owned_records(res, record_name, alias_dns):
    return [dict(name=record_name, type="TXT", values=[owner_value(res)]), dict(name=record_name, type="A", alias=alias_dns + ".")]


def owning_world(owners, extra_objects=(), cached=None):
    """objects of kind/key `owners` (in this row order); each owns one accelerator (list order = owners order), and in zone
    example.com. the TXT owner value and the A alias of its hostname.  `cached`: the owners that are objects of the cache (the
    others left it: their resources are orphans).  Returns (objects, actual)."""
    objects, accs, recs, lbs = [], [], [], []
    for i, (kind, key) in enumerate(owners):
        name = f"lb{i:02d}"
        lbs.append(lb(name, i))
        ob = obj(kind, key, lb_host(name), r53=f"h{i}.example.com")
        a = accel(i, resource(ob), lb_host(name), lbs[-1]["arn"], name="stale" if i % 2 else f"{kind}-{key.replace('/', '-')}")
        accs.append(a)
        recs += owned_records(resource(ob), f"h{i}.example.com.", a["dns"] if i % 3 else "stale.awsglobalaccelerator.com")
        if cached is None or i in cached:
            objects.append(ob)
    objects += list(extra_objects)
    return objects, dict(lbs=lbs, accelerators=accs, zones=[dict(id="/hostedzone/Z0", name="example.com.", records=recs)])


def check_all(garecon, oracle, e, objects, actual, rows, deleted=(), bindings=None):
    """gar_diff_keys (before any full diff: the indexes are built on demand), gar_diff, gar_diff_keys again, and
    gar_bindings_diff, each equal to the oracle bit for bit.  Returns the packed snapshot: the host simulation reads its buffers
    for as long as it is loaded."""
    snap = garecon.pack(objects, actual)
    e.load(snap)
    for step in ("keys", "full", "keys"):
        if step == "keys":
            got, want = e.diff_keys(rows, list(deleted)), oracle.diff_keys(snap, rows, list(deleted), mode=1)
        else:
            got, want = e.diff(), oracle.diff(snap, "default", mode=1)
        assert got.diff(want) == [], f"{step}: {got.describe_first_mismatch(want)}"
    if bindings is not None:
        got, want = e.bindings_diff(bindings), oracle.bindings_diff(snap, bindings)
        assert got.diff(want) == [], f"bindings: {got.describe_first_mismatch(want)}"
    return snap


def kinded_hash(kind, key):
    return C.key_hash_kinded(0 if kind == "service" else 1, key)


def assert_object_collisions(pairs, objects, actual, bits=BITS):
    rows = C.table_rows(objects, actual)
    for (ka, a), (kb, b) in pairs:
        ha, hb = kinded_hash(ka, a), kinded_hash(kb, b)
        for index in ("obj", "owner", "val"):
            C.assert_collide(ha, hb, index, rows[index], bits)


# ------------------------------------------------------------------ 1. objects: ix_obj, canon_bucket, owned lists

def scenario_objects(garecon, oracle, make_engine, placement):
    """ix_obj probes (find_object in the value pass, the egb ref lookup), canon_bucket (which rows repeat a key) and the owned
    lists built from them: two Services whose keys collide, a Service / Ingress pair that collides across kinds, one key that
    is both a Service and an Ingress (tag and bucket equal: only the kind tells them apart), and a genuinely repeated key placed
    after its colliding impostor.  Each object's ops must come from its own accelerators and owner values."""
    tpl = C.OBJECT_KEYS[placement]
    a, b = pair(C.kinded_fn(0), tpl, placement)
    s, i = pair(C.kinded_fn(0), tpl, placement, seed=1, fn_b=C.kinded_fn(1))
    same = C.SAME_KEY_BOTH_KINDS
    owners = [("service", b), ("service", a), ("ingress", i), ("service", s), ("ingress", same), ("service", same)]
    objects, actual = owning_world(owners)
    objects.append(copy.deepcopy(objects[1]))  # the key of row 1 again, after its impostor at row 0
    assert_object_collisions([(("service", a), ("service", b)), (("service", s), ("ingress", i))], objects, actual)
    assert_object_collisions([(("service", same), ("ingress", same))], objects, actual, bits=C.SAME_KEY_BITS)
    eg = "arn:aws:globalaccelerator::1:accelerator/x/listener/0/endpoint-group/0"
    bindings = [dict(ns=key.split("/", 1)[0], ref=(kind, key.split("/", 1)[1]), eg_arn=eg, deleting=False, finalizers=True, observed=True,
                     endpoint_ids=[]) for kind, key in owners[1:]]  # every ref but the lowest row's has a colliding key at a lower row
    with make_engine() as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=list(range(len(objects))), bindings=garecon.pack_bindings(bindings, [eg]))
        got = e.diff()
    ga = got.ops[:int(got.section_begin[1])]
    acc_of = lambda r: sorted({int(op["a0"]) for op in ga if op["obj"] == r})  # noqa: E731
    assert acc_of(1) and acc_of(len(objects) - 1) == acc_of(1)  # the repeated key reads its own first row's lists


# ------------------------------------------------------------------ 2. orphans through a collision

def scenario_orphans(garecon, oracle, make_engine, placement):
    """resolve_accel / resolve_value (find_object) for resources of a key that left the cache while its collider is in it: B's
    accelerator and owner values land in the GA and Route53 orphan sections, A's are untouched.  With orphans=False the orphan
    sections stay empty and the object sections are unchanged."""
    a, b = pair(C.kinded_fn(0), C.OBJECT_KEYS[placement], placement)
    objects, actual = owning_world([("service", b), ("service", a)], cached={1})
    assert_object_collisions([(("service", a), ("service", b))], objects, actual)
    with make_engine() as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=[0], deleted=[(0, b)])
        got = e.diff()
    sb = [int(x) for x in got.section_begin]
    assert [int(op["a0"]) for op in got.ops[sb[1]:sb[2]]][:1] == [0]  # B's accelerator (row 0) is deleted as an orphan
    assert sb[4] > sb[3]
    want = oracle.diff(garecon.pack(objects, actual), "default", mode=1)
    with make_engine(orphans=False) as e:
        snap = garecon.pack(objects, actual)
        e.load(snap)
        got = e.diff()
    gb = [int(x) for x in got.section_begin]
    assert gb[2] == gb[1] and gb[4] == gb[3]
    assert np.array_equal(got.ops[gb[0]:gb[1]], want.ops[sb[0]:sb[1]]) and np.array_equal(got.ops[gb[2]:gb[3]], want.ops[sb[2]:sb[3]])
    assert np.array_equal(got.status_ga, want.status_ga) and np.array_equal(got.status_r53, want.status_r53)


# ------------------------------------------------------------------ 3. load balancers: ix_lb

def scenario_load_balancers(garecon, oracle, make_engine, placement):
    """find_lb (bindings, diff_keys) and u_find_lb (the GA pass): two (region, name) keys collide; the impostor is listed first
    and is still provisioning, so a wrong pick changes the status word and the endpoint ARN."""
    real, fake = pair(C.lb_fn(REGION), LB_NAMES[placement], placement)
    lbs = [lb(fake, 1, state="provisioning"), lb(real, 2)]
    objects = [obj("service", "default/web", lb_host(real)), obj("service", "default/other", lb_host(fake))]
    accs = [accel(0, "service/default/web", lb_host(real), lbs[1]["arn"], name="stale"), accel(1, "service/default/other", lb_host(fake), lbs[0]["arn"])]
    actual = dict(lbs=lbs, accelerators=accs, zones=[])
    C.assert_collide(C.key_hash_lb(REGION, real), C.key_hash_lb(REGION, fake), "lb", len(lbs), BITS)
    eg = "arn:aws:globalaccelerator::1:accelerator/x/listener/0/endpoint-group/0"
    bindings = [dict(ns="default", ref=("service", "web"), eg_arn=eg, deleting=False, finalizers=True, observed=True, endpoint_ids=[]),
                dict(ns="default", ref=("service", "other"), eg_arn=eg, deleting=False, finalizers=True, observed=True, endpoint_ids=[lbs[0]["arn"]])]
    with make_engine() as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=[0, 1], bindings=garecon.pack_bindings(bindings, [eg]))


# ------------------------------------------------------------------ 4. target hostnames: ix_thost

def thost_world(placement):
    real, fake = pair(C.hash_matrix, THOSTS[placement], placement)
    objects = [obj("service", "default/imp", fake, r53="imp.example.com"), obj("service", "default/web", real, r53="web.example.com")]
    # two accelerators carry the colliding hostname ahead of the real one: a walk that stops after two matches (the sharded
    # answer pass, gar_shard.h) never reaches the real accelerator unless it compares keys
    accs = [accel(0, "service/default/imp", fake), accel(2, "service/default/imp", fake), accel(1, "service/default/web", real)]
    recs = owned_records("service/default/web", "web.example.com.", accs[2]["dns"]) + owned_records("service/default/imp", "imp.example.com.", "stale.x")
    actual = dict(lbs=[], accelerators=accs, zones=[dict(id="/hostedzone/Z0", name="example.com.", records=recs)])
    C.assert_collide(C.key_hash_str(real), C.key_hash_str(fake), "thost", len(accs), BITS)
    return objects, actual


def scenario_target_hostnames(garecon, oracle, make_engine, placement):
    """find_by_hostname / u_find_by_hostname (Route53 by lbIngress hostname): an accelerator tagged with a colliding hostname is
    listed before the real one; counted as a match it would flip the "more than one accelerator" path."""
    objects, actual = thost_world(placement)
    with make_engine() as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=[0, 1])


# ------------------------------------------------------------------ 5. hosted zones: ix_zone

def scenario_hosted_zones(garecon, oracle, make_engine, placement):
    """find_hosted_zone / u_find_hosted_zone: the hostname's zone collides with another zone name of the same length (so both
    pass zone_len_possible), listed first."""
    real, fake = pair(C.hash_matrix, ZONE_NAMES[placement], placement)
    objects = [obj("service", "default/web", lb_host("web"), r53=f"app.{real}"), obj("service", "default/imp", lb_host("imp"), r53=f"app.{fake}")]
    accs = [accel(0, "service/default/web", lb_host("web")), accel(1, "service/default/imp", lb_host("imp"))]
    zones = [dict(id="/hostedzone/ZF", name=fake + ".", records=owned_records("service/default/imp", f"app.{fake}.", "stale.x")),
             dict(id="/hostedzone/ZR", name=real + ".", records=owned_records("service/default/web", f"app.{real}.", accs[0]["dns"]))]
    actual = dict(lbs=[], accelerators=accs, zones=zones)
    assert len(real) == len(fake)
    C.assert_collide(C.key_hash_str(real), C.key_hash_str(fake), "zone", len(zones), BITS)
    with make_engine() as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=[0, 1])


# ------------------------------------------------------------------ 6. aliases and orphan values: ix_alias, ix_ovn

def alias_world(placement, two_hosts=False):
    """two_hosts: every object has two lbIngress hostnames, each with its own accelerator, so that Route53 evaluates it per object
    (r53_reconcile, which finds the alias record with u_first_alias_a) instead of per (object, hostname) pair"""
    real, fake = pair(C.zoned_fn(0), RECORD_NAMES[placement], placement)
    objects = [obj("service", "default/web", lb_host("web"), r53=real[:-1]), obj("service", "default/imp", lb_host("imp"), r53=fake[:-1])]
    accs = [accel(0, "service/default/web", lb_host("web")), accel(1, "service/default/imp", lb_host("imp"))]
    if two_hosts:
        for k, ob in enumerate(objects):
            ob["lb_ingress"].append(lb_host(ob["name"] + "2"))
            accs.append(accel(2 + k, resource(ob), lb_host(ob["name"] + "2")))
    gone = owner_value("service/default/gone")
    # one of the two aliases is in sync with web's accelerator and the other is not, so a lookup for web's name that takes the
    # impostor's record changes web's ops: the impostor's is stale in the first model, web's own in the second
    good, stale = accs[0]["dns"] + ".", "stale.awsglobalaccelerator.com."
    recs = [dict(name=fake, type="TXT", values=[owner_value("service/default/imp"), gone]), dict(name=fake, type="A", alias=good if two_hosts else stale),
            dict(name=real, type="TXT", values=[owner_value("service/default/web"), gone]), dict(name=real, type="A", alias=stale if two_hosts else good)]
    actual = dict(lbs=[], accelerators=accs, zones=[dict(id="/hostedzone/Z0", name="example.com.", records=recs)])
    rows = C.table_rows(objects, actual)
    for index in ("alias", "ovn"):
        C.assert_collide(C.key_hash_zoned(0, real), C.key_hash_zoned(0, fake), index, rows[index], BITS)
    return objects, actual


def scenario_aliases(garecon, oracle, make_engine, placement):
    """first_alias_a / next_alias_any and the ix_ovn walk with its duplicate check (r53_orphan_alias): two record names of one
    zone collide; each carries an A alias, its owner's value and the same orphan owner value.  The second model gives every
    object two lbIngress hostnames, which takes Route53 through r53_reconcile and its u_first_alias_a."""
    for two_hosts in (False, True):
        objects, actual = alias_world(placement, two_hosts)
        with make_engine() as e:
            snap = check_all(garecon, oracle, e, objects, actual, rows=[0, 1], deleted=[(0, "default/gone")])


# ------------------------------------------------------------------ 7. deleted keys: ix_owner, ix_val

def scenario_deleted_keys(garecon, oracle, make_engine, placement):
    """owner_next and owned_collect / owned_get (built on demand for deleted keys): a deleted key whose collider is in the cache
    and owns resources, and the reverse, before and after a full diff."""
    a, b = pair(C.kinded_fn(0), C.OBJECT_KEYS[placement], placement)
    for cached, gone in ((1, b), (0, a)):
        objects, actual = owning_world([("service", b), ("service", a)], cached={cached})
        assert_object_collisions([(("service", a), ("service", b))], objects, actual)
        with make_engine() as e:
            snap = check_all(garecon, oracle, e, objects, actual, rows=[0], deleted=[(0, gone)])


# ------------------------------------------------------------------ 8. bindings: ix_eg

def scenario_bindings(garecon, oracle, make_engine, placement):
    """egb_eg_exists: known endpoint-group ARNs that collide with a binding's ARN are not that ARN."""
    real, fake = pair(C.hash_matrix, EG_ARN, "tail")
    objects, actual = owning_world([("service", "default/web")])
    base = dict(ns="default", ref=("service", "web"), finalizers=True, observed=True)
    bindings = [dict(base, eg_arn=real, deleting=True, endpoint_ids=[actual["lbs"][0]["arn"]]),
                dict(base, eg_arn=real, deleting=False, endpoint_ids=[]),
                dict(base, eg_arn=fake, deleting=True, endpoint_ids=[actual["lbs"][0]["arn"]])]
    known = [fake]
    C.assert_collide(C.key_hash_str(real), C.key_hash_str(fake), "eg", len(known), BITS)
    with make_engine() as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=[0], bindings=garecon.pack_bindings(bindings, known))


# ------------------------------------------------------------------ 9. object deltas: the gar_delta.h key resolver

def scenario_object_deltas(garecon, oracle, make_engine, placement):
    """FDeltaResolve: with A resident, deleting its collider B finds nothing, upserting B appends a row and leaves A's alone,
    and deleting A leaves B.  After every step the diffs equal the oracle on the table the delta rules prescribe."""
    a, b = pair(C.kinded_fn(0), C.OBJECT_KEYS[placement], placement)
    objects, actual = owning_world([("service", b), ("service", a)], cached={1})
    objects.append(obj("service", "default/filler", lb_host("filler")))
    ob_b = owning_world([("service", b)])[0][0]
    assert_object_collisions([(("service", a), ("service", b))], objects + [ob_b], actual)
    snap = garecon.pack(objects, actual)
    with make_engine() as e:
        e.load(snap)
        e.diff()
        m = Mirror(objects, snap)
        for upserts, deleted in (([], [(0, b)]), ([ob_b], []), ([], [(0, a)]), ([], [(0, a)])):
            usnap = garecon.pack(upserts, None) if upserts else None
            res = e.apply_objects(usnap.objects if usnap else None, deleted)
            up_row, del_row, moved, _ = m.apply(upserts, deleted, usnap)
            assert (res.upsert_row.tolist(), res.deleted_row.tolist(), res.moved_from.tolist()) == (up_row, del_row, moved)
            msnap = garecon.pack(m.objects, actual)
            rows = list(range(len(m.objects)))
            got, want = e.diff_keys(rows, [(0, a), (0, b)]), oracle.diff_keys(msnap, rows, [(0, a), (0, b)], mode=1)
            assert got.diff(want) == [], got.describe_first_mismatch(want)
            assert_same_full(e.diff(), oracle.diff(msnap, "default", mode=1), m.slab, msnap.arrays["o.slab"])
        assert sorted(key_of(o) for o in m.objects) == sorted([(0, "default/filler"), (0, b)])


# ------------------------------------------------------------------ 10. the radix fallback

def radix_world(placement):
    a, b = pair(C.kinded_fn(0), C.OBJECT_KEYS[placement], placement)
    owners = [("service", b), ("service", a)] * 50  # 50 rows of each key in one ix_obj bucket, each row owning an accelerator and a value
    objects, actual = owning_world(owners)
    assert_object_collisions([(("service", a), ("service", b))], objects, actual)
    return objects, actual


def scenario_radix(garecon, oracle, make_engine, placement):
    """More than IDX_SMALL_BUCKET (48) rows in one bucket, mixing two tag-colliding keys with true duplicates of each: ix_obj goes
    through the stable radix build (FIdxGather, FIdxCanon) and the owned lists of both keys (50 accelerators and values) through
    the radix path of the list build."""
    objects, actual = radix_world(placement)
    with make_engine() as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=[0, 1, len(objects) - 2, len(objects) - 1])


# ------------------------------------------------------------------ 11. warp placement (GPU)

WARP_ROWS = (0, 31, 255, 256)  # lanes 0 and 31 of the first warp, and both sides of the first 256-row block boundary


def warp_world(n_objects=300):
    """n_objects Services, every one with two lbIngress hostnames (Route53 per object: u_find_by_hostname, u_find_hosted_zone and
    u_first_alias_a in r53_reconcile; u_find_lb in the GA pass).  The objects at WARP_ROWS probe colliding keys: an LB name, a
    target hostname, a hosted zone and an alias record name, each with its impostor listed first.  Every other object probes
    plain keys shared by groups of objects, so the voted bucket walks of a warp mix tag hits that fail the key compare with
    ordinary hits and misses.  The AWS tables stay within 2**BITS buckets (asserted); the object table does not need to."""
    k = len(WARP_ROWS)
    lb_pairs = C.find_pairs(C.lb_fn(REGION), LB_NAMES["tail"], k, bits=BITS, seed=7)
    host_pairs = C.find_pairs(C.hash_matrix, THOSTS["middle"], k, bits=BITS, seed=7)
    zone_pairs = C.find_pairs(C.hash_matrix, ZONE_NAMES["first"], k, bits=BITS, seed=7)
    name_pairs = C.find_pairs(C.zoned_fn(0), RECORD_NAMES["first"], k, bits=BITS, seed=7)
    lbs, accs, objects = [], [], []
    zones = [dict(id="/hostedzone/Z0", name="example.com.", records=[])] + [dict(id=f"/hostedzone/ZF{j}", name=f + ".", records=[]) for j, (_, f) in enumerate(zone_pairs)]
    zones += [dict(id=f"/hostedzone/ZR{j}", name=r + ".", records=[]) for j, (r, _) in enumerate(zone_pairs)]
    recs = zones[0]["records"]
    plain = [(lb_host(f"plain{g}a"), lb_host(f"plain{g}b")) for g in range(8)]
    for g, hosts in enumerate(plain):
        for h in hosts:
            lbs.append(lb(h.split("-")[0], len(lbs)))
            accs.append(accel(len(accs), f"service/default/group{g}", h, lbs[-1]["arn"]))
    for j, r in enumerate(WARP_ROWS):
        (lb_real, lb_fake), (h_real, h_fake), (z_real, _), (n_real, n_fake) = lb_pairs[j], host_pairs[j], zone_pairs[j], name_pairs[j]
        lbs += [lb(lb_fake, len(lbs), state="provisioning"), lb(lb_real, len(lbs) + 1), lb(h_real.split("-0123")[0], len(lbs) + 2)]
        res = f"service/default/o{r}"
        accs += [accel(len(accs), "service/default/nobody", h_fake), accel(len(accs) + 1, res, h_real, lbs[-1]["arn"]),
                 accel(len(accs) + 2, res, lb_host(lb_real), lbs[-2]["arn"])]
        recs += [dict(name=n_fake, type="TXT", values=[owner_value("service/default/nobody")]), dict(name=n_fake, type="A", alias=accs[-2]["dns"] + "."),
                 dict(name=n_real, type="TXT", values=[owner_value(res)]), dict(name=n_real, type="A", alias="stale.awsglobalaccelerator.com.")]
        zones[1 + k + j]["records"] += owned_records(res, f"app.{z_real}.", accs[-2]["dns"])
    special = {r: j for j, r in enumerate(WARP_ROWS)}
    for i in range(n_objects):
        if i in special:
            j = special[i]
            ob = obj("service", f"default/o{i}", host_pairs[j][0], r53=f"{name_pairs[j][0][:-1]},app.{zone_pairs[j][0]}")
            ob["lb_ingress"].append(lb_host(lb_pairs[j][0]))
        else:
            ob = obj("service", f"default/o{i}", plain[i % 8][0], r53=f"p{i}.example.com")
            ob["lb_ingress"].append(plain[i % 8][1])
            if i % 3 == 0:  # a third of the plain objects own their record (an alias lookup that hits)
                recs += owned_records(resource(ob), f"p{i}.example.com.", accs[2 * (i % 8)]["dns"] if i % 2 else "stale.awsglobalaccelerator.com")
        objects.append(ob)
    actual = dict(lbs=lbs, accelerators=accs, zones=zones)
    rows = C.table_rows(objects, actual)
    for j in range(k):
        C.assert_collide(C.key_hash_lb(REGION, lb_pairs[j][0]), C.key_hash_lb(REGION, lb_pairs[j][1]), "lb", rows["lb"], BITS)
        C.assert_collide(C.key_hash_str(host_pairs[j][0]), C.key_hash_str(host_pairs[j][1]), "thost", rows["thost"], BITS)
        C.assert_collide(C.key_hash_str(zone_pairs[j][0]), C.key_hash_str(zone_pairs[j][1]), "zone", rows["zone"], BITS)
        C.assert_collide(C.key_hash_zoned(0, name_pairs[j][0]), C.key_hash_zoned(0, name_pairs[j][1]), "alias", rows["alias"], BITS)
    return objects, actual


def scenario_warp_placement(garecon, oracle, make_engine):
    """the voted U_BUCKET_LOOP walks of u_find_lb, u_find_by_hostname, u_find_hosted_zone and u_first_alias_a with colliding
    probes at lanes 0 and 31 of a warp and on both sides of a 256-row block boundary, the other lanes probing plain keys"""
    objects, actual = warp_world()
    with make_engine() as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=list(range(len(objects))))
        snap = check_all(garecon, oracle, e, objects, actual, rows=[250, 255, 256, 31, 0, 7])


SCENARIOS = {"objects": scenario_objects, "orphans": scenario_orphans, "load_balancers": scenario_load_balancers,
             "deleted_keys": scenario_deleted_keys, "object_deltas": scenario_object_deltas, "radix": scenario_radix}
# scenarios whose keys cannot take every placement (hostnames keep their DNS suffix, record names their zone)
TWO_PLACEMENTS = {"target_hostnames": scenario_target_hostnames, "aliases": scenario_aliases}
ONE_PLACEMENT = {"hosted_zones": scenario_hosted_zones, "bindings": scenario_bindings}


def all_cases():
    cases = [(n, p) for n in sorted(SCENARIOS) for p in C.PLACEMENTS]
    cases += [(n, p) for n in sorted(TWO_PLACEMENTS) for p in ("first", "middle")]
    cases += [(n, p) for n in sorted(ONE_PLACEMENT) for p in (C.PLACEMENTS if n == "hosted_zones" else ["tail"])]
    return cases


def run_case(garecon, oracle, make_engine, name, placement):
    fn = SCENARIOS.get(name) or TWO_PLACEMENTS.get(name) or ONE_PLACEMENT[name]
    fn(garecon, oracle, make_engine, placement)


@pytest.fixture(scope="module")
def hostlib(garecon):
    import __graft_entry__ as ge
    return garecon.abi.load_library(ge.build_hostsim())


@pytest.mark.parametrize("name,placement", all_cases())
def test_hostsim_collisions(garecon, oracle, hostlib, name, placement):
    run_case(garecon, oracle, lambda **kw: garecon.Engine(cluster_name="default", lib=hostlib, **kw), name, placement)


def test_hostsim_warp_placement(garecon, oracle, hostlib):
    """the warp-placement model on the host simulation (its 32 host threads emulate a warp's votes)"""
    scenario_warp_placement(garecon, oracle, lambda **kw: garecon.Engine(cluster_name="default", lib=hostlib, **kw))


# ------------------------------------------------------------------ 12. sharded (host simulation)

@pytest.mark.parametrize("world", ["target_hostnames", "aliases"])
@pytest.mark.parametrize("placement", ["first", "middle"])
def test_hostsim_sharded_collisions(garecon, oracle, hostlib, world, placement):
    """the sharded alias and hostname marks (gar_shard.h) over the colliding models of scenarios 4 and 6, split over 2 ranks:
    the merged change set equals the unsharded one and the oracle.  The hostname answer pass (FShAnswer) stops after two
    matches, and the hostname model puts two colliding accelerators ahead of the real one: without its key compare the real
    accelerator never reaches the probe's shard.  The alias mark (FShRecMask) is only exercised: an impostor record it marked
    wrongly would merely be copied to one more shard, where no lookup matches it."""
    from test_sharded import check
    objects, actual = (thost_world if world == "target_hostnames" else alias_world)(placement)
    got, _ = check(garecon, oracle, hostlib, objects, actual, 2)
    with garecon.Engine(cluster_name="default", lib=hostlib) as e:
        snap = garecon.pack(objects, actual)
        e.load(snap)
        assert got["ops"].tolist() == e.diff().ops.tolist()


# ------------------------------------------------------------------ the mirror is the device hash

PIN_SRC = textwrap.dedent(r'''
    #include <stdio.h>
    #include <stdlib.h>
    #include <string.h>
    #include "gar_rows.h"
    bool gar_host_vote(bool p) { return p; }  // one lane: every vote is that lane's own predicate
    static int hexval(int c) { return c <= '9' ? c - '0' : c - 'a' + 10; }
    int main() {
      static char line[1 << 12];
      alignas(16) static u8 buf[1 << 11], prev[1 << 11];
      u32 pn = 0, lineno = 0;
      while (fgets(line, sizeof line, stdin)) {
        u32 n = (u32)(strcspn(line, "\n") / 2);
        lineno++;
        for (u32 i = 0; i < sizeof buf; i++) buf[i] = (u8)(lineno + i);  // bytes past the end differ from the previous key's
        for (u32 i = 0; i < n; i++) buf[i] = (u8)(hexval(line[2 * i]) * 16 + hexval(line[2 * i + 1]));
        Str s{buf, n}, p{prev, pn};
        printf("%016llx %016llx %016llx %016llx %016llx %016llx %016llx %d\n", (unsigned long long)gar_hash(s), (unsigned long long)u_hash(true, s),
               (unsigned long long)key_hash_kinded(0, s), (unsigned long long)key_hash_kinded(1, s), (unsigned long long)key_hash_zoned(3, s),
               (unsigned long long)key_hash_lb(p, s), (unsigned long long)key_hash_str(s), (int)u_streq(true, s, p));
        memcpy(prev, buf, sizeof buf);
        pn = n;
      }
      return 0;
    }
''')


def pinned_strings():
    rng = np.random.default_rng(5)
    out = [b"", b"a", b"default/svc-2aqwa", b"default/svc-nvd3b", C.SAME_KEY_BOTH_KINDS.encode()]
    for _ in range(1000):
        n = int(rng.integers(0, 41))
        out.append(bytes(rng.integers(0, 256, n, dtype=np.uint8)) if rng.random() < 0.3 else bytes(rng.choice(list(C.ALPHABET + b"/.-"), n).astype(np.uint8)))
    for s in range(2):  # keys that differ only in the masked tail word, and a key compared with itself
        for a, b in C.find_pairs(C.kinded_fn(0), C.OBJECT_KEYS["tail"], 1, bits=BITS, seed=s):
            out += [a.encode(), b.encode(), b.encode()]
    return out


def scenario_keys():
    keys = []
    for p in C.PLACEMENTS:
        keys += pair(C.kinded_fn(0), C.OBJECT_KEYS[p], p) + pair(C.kinded_fn(0), C.OBJECT_KEYS[p], p, seed=1, fn_b=C.kinded_fn(1))
        keys += pair(C.lb_fn(REGION), LB_NAMES[p], p) + pair(C.hash_matrix, ZONE_NAMES[p], p)
    for p in ("first", "middle"):
        keys += pair(C.hash_matrix, THOSTS[p], p) + pair(C.zoned_fn(0), RECORD_NAMES[p], p)
    keys += pair(C.hash_matrix, EG_ARN, "tail")
    return [k.encode() for k in keys]


def test_mirror_matches_the_device_hashes(tmp_path):
    """every key_hash_* of csrc/gar_rows.h (compiled with g++) equals the numpy mirror bit for bit, for random strings of 0..40
    bytes (bytes >= 0x80 included) and for every key the scenarios use; u_hash equals gar_hash and u_streq is byte-exact"""
    (tmp_path / "pin.cpp").write_text(PIN_SRC)
    exe = tmp_path / "pin"
    subprocess.run(["g++", "-O1", "-std=c++17", "-w", "-I", str(CSRC), "-o", str(exe), str(tmp_path / "pin.cpp")], check=True)
    strings = pinned_strings() + scenario_keys()
    out = subprocess.run([str(exe)], input="".join(s.hex() + "\n" for s in strings), capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(out) == len(strings)
    prev = b""
    for s, line in zip(strings, out):
        f = line.split()
        got = [int(x, 16) for x in f[:7]]
        want = [C.gar_hash(s), C.gar_hash(s), C.key_hash_kinded(0, s), C.key_hash_kinded(1, s), C.key_hash_zoned(3, s), C.key_hash_lb(prev, s), C.key_hash_str(s)]
        assert got == want, s
        assert int(f[7]) == int(s == prev), s
        prev = s
    h0, h1 = C.key_hash_kinded(0, C.SAME_KEY_BOTH_KINDS), C.key_hash_kinded(1, C.SAME_KEY_BOTH_KINDS)
    assert C.tag(h0) == C.tag(h1) and C.bucket(h0, 1 << C.SAME_KEY_BITS) == C.bucket(h1, 1 << C.SAME_KEY_BITS)


def test_pairs_are_deterministic_and_distinct():
    a = C.find_pairs(C.kinded_fn(0), "default/svc-{}", 2, bits=BITS, seed=3, free=5)
    C._search.cache_clear()
    assert C.find_pairs(C.kinded_fn(0), "default/svc-{}", 2, bits=BITS, seed=3, free=5) == a
    assert len({k for p in a for k in p}) == 4
    for x, y in a:
        C.assert_collide(C.key_hash_kinded(0, x), C.key_hash_kinded(0, y), "obj", 1 << BITS, BITS)


# ------------------------------------------------------------------ GPU tier

@pytest.mark.gpu
@pytest.mark.parametrize("name,placement", all_cases())
def test_gpu_collisions(garecon, oracle, name, placement):
    import __graft_entry__ as ge
    ge.ensure_built()
    run_case(garecon, oracle, lambda **kw: garecon.Engine(cluster_name="default", device=0, **kw), name, placement)


@pytest.mark.gpu
def test_gpu_radix_fallback_runs(garecon, oracle):
    """the radix scenario really takes the stable radix sort on the device"""
    objects, actual = radix_world("tail")
    with garecon.Engine(cluster_name="default", device=0, stage_timing=True) as e:
        snap = check_all(garecon, oracle, e, objects, actual, rows=[0, 1])
        e.load(snap)  # the timings are those of the last call: a full diff that builds every index from scratch
        e.diff()
        assert "radix_sort_pairs" in {s[0] for s in e.stage_timings()}


@pytest.mark.gpu
def test_gpu_warp_placement(garecon, oracle):
    import __graft_entry__ as ge
    ge.ensure_built()
    scenario_warp_placement(garecon, oracle, lambda **kw: garecon.Engine(cluster_name="default", device=0, **kw))
