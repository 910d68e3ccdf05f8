"""The per-lbIngress-row lookups (Work::lbi_res, gar_rows.h lbi_resolve): every row's load balancer with its verdict, and the
accelerators whose target-hostname tag equals the row's hostname, resolved once and read by the Global Accelerator and Route53
decisions.  The record depends on both sides of the snapshot, so it must be rebuilt after every change to either: object deltas
(rows repointed, lbIngress rows shifted), AWS deltas (the matched LB deleted, its DNS name re-described, its state flipped; a
second accelerator with the same target hostname), zone deltas and the compaction of each slab group.  After each change
gar_diff_keys and a full diff (the snapshot prepared once, not every diff) must equal the oracle on the changed model.  The world
also holds a load balancer whose (region, name) collides in bucket and tag with an impostor listed first, a target hostname that
collides with another accelerator's tag, and an object with two lbIngress rows whose second load balancer differs.

Every array of the change set is compared bit for bit except tok_name / tok_region: those are references into the object slab,
which deltas and the compaction move, and the tokeniser that writes them is not what this file tests."""
import pytest

import collisions as C
from test_hash_collisions import LB_NAMES, REGION, THOSTS, accel, lb, lb_host, obj, owned_records, pair
from test_zone_deltas import State

NONE = 0xFFFFFFFF
COMPARED = ("status_ga", "status_r53", "derived", "ops", "section_begin", "tok_code", "dport_begin", "dports")


def world():
    """(objects, actual): six objects over seven load balancers and eight accelerators, each object owning its accelerator"""
    real, fake = pair(C.lb_fn(REGION), LB_NAMES["tail"], "tail")
    h_real, h_fake = pair(C.hash_matrix, THOSTS["middle"], "middle")
    names = [fake, "web", "api", "alt", real, h_real.split("-0123")[0], "ing"]
    lbs = [lb(n, i, state="provisioning" if n == fake else "active") for i, n in enumerate(names)]
    arn = {n: x["arn"] for n, x in zip(names, lbs)}
    assert lb_host(names[5]) == h_real
    objects = [obj("service", "default/web", lb_host("web"), r53="web.example.com"),
               obj("service", "default/api", lb_host("api"), r53="api.example.com"),
               obj("service", "default/multi", lb_host("web"), r53="multi.example.com"),
               obj("service", "default/coll", lb_host(real), r53="coll.example.com"),
               obj("service", "default/thost", h_real, r53="th.example.com"),
               obj("ingress", "default/ing", lb_host("ing"))]
    objects[2]["lb_ingress"].append(lb_host("alt"))  # the self-observation path: a second lbIngress with another load balancer
    accs = [accel(0, "service/default/nobody", h_fake),  # the colliding target hostname, listed ahead of the real one
            accel(1, "service/default/web", lb_host("web"), arn["web"]),
            accel(2, "service/default/api", lb_host("api"), arn["api"], name="service-default-api"),
            accel(3, "service/default/multi", lb_host("web"), arn["web"]),
            accel(4, "service/default/coll", lb_host(real), arn[real]),
            accel(5, "service/default/thost", h_real, arn[names[5]]),
            accel(6, "ingress/default/ing", lb_host("ing"), arn["ing"]),
            accel(7, "service/default/gone", lb_host("alt"), arn["alt"])]
    recs = owned_records("service/default/web", "web.example.com.", accs[1]["dns"]) + owned_records("service/default/api", "api.example.com.", "stale.x")
    recs += owned_records("service/default/thost", "th.example.com.", accs[5]["dns"])
    actual = dict(lbs=lbs, accelerators=accs, zones=[dict(id="/hostedzone/Z0", name="example.com.", records=recs)])
    rows = C.table_rows(objects, actual)
    C.assert_collide(C.key_hash_lb(REGION, real), C.key_hash_lb(REGION, fake), "lb", rows["lb"], 8)
    C.assert_collide(C.key_hash_str(h_real), C.key_hash_str(h_fake), "thost", rows["thost"], 8)
    return objects, actual


def same(got, want, what):
    bad = [k for k in COMPARED if getattr(got, k).shape != getattr(want, k).shape or (getattr(got, k) != getattr(want, k)).any()]
    assert not bad, f"{what}: {bad}: {got.describe_first_mismatch(want)}"


def check(st, what):
    """gar_diff_keys over every row (the first diff after the change: it rebuilds what the change made stale), then a full diff"""
    msnap = st.msnap()
    rows = list(range(len(st.om.objects)))
    same(st.e.diff_keys(rows, []), st.oracle.diff_keys(msnap, rows, [], mode=1), f"{what}: diff_keys")
    same(st.e.diff(), st.oracle.diff(msnap, "default", mode=1), f"{what}: full diff")


def upsert(st, ob):
    usnap = st.g.pack([ob], None)
    st.e.apply_objects(usnap.objects, [])
    st.om.apply([ob], [], usnap)


def lb_row(st, name):
    return next(r for r, x in enumerate(st.model.actual["lbs"]) if x["name"] == name)


def run(garecon, oracle, make_engine):
    objects, actual = world()
    with make_engine() as e:
        st = State(garecon, oracle, e, objects, actual)
        check(st, "load")
        upsert(st, obj("service", "default/api", lb_host("alt"), r53="api.example.com"))  # repointed at another LB
        check(st, "object delta: lbIngress hostname repointed")
        web = obj("service", "default/web", lb_host("ing"), r53="web.example.com")
        web["lb_ingress"].append(lb_host("web"))  # a row ahead of the object's old one: every later lbIngress row shifts
        upsert(st, web)
        check(st, "object delta: lbIngress rows shifted")
        st.aws({"lb_deleted": [lb_row(st, "web")]})
        check(st, "AWS delta: matched load balancer deleted")
        alt = st.model.actual["lbs"][lb_row(st, "alt")]
        st.aws({"lbs": [(lb_row(st, "alt"), dict(alt, dns="re-described.elb.us-east-1.amazonaws.com"))]})
        check(st, "AWS delta: DNS name re-described")
        st.aws({"lbs": [(lb_row(st, "alt"), dict(alt, state="provisioning"))]})
        check(st, "AWS delta: state active -> provisioning")
        st.aws({"lbs": [(lb_row(st, "alt"), dict(alt, state="active"))]})
        check(st, "AWS delta: state provisioning -> active")
        st.aws({"accs": [(NONE, accel(8, "service/default/other", lb_host("ing")))]})
        check(st, "AWS delta: a second accelerator with the same target hostname")
        st.zones(added=[(0, dict(id="/hostedzone/Z1", name="api.example.com.", records=[]))])
        check(st, "zone delta")
        e.compact(garecon.abi.COMPACT_OBJECTS)
        check(st, "compaction of the object slab")
        e.compact(garecon.abi.COMPACT_ACTUAL)
        check(st, "compaction of the AWS slab")
        upsert(st, obj("service", "default/coll", lb_host("alt"), r53="coll.example.com"))
        check(st, "object delta after both compactions")


@pytest.fixture(scope="module")
def hostlib(garecon):
    import __graft_entry__ as ge
    return garecon.abi.load_library(ge.build_hostsim())


def test_hostsim_lbi_records_follow_every_state_change(garecon, oracle, hostlib):
    run(garecon, oracle, lambda: garecon.Engine(cluster_name="default", lib=hostlib))


@pytest.mark.gpu
def test_gpu_lbi_records_follow_every_state_change(garecon, oracle):
    run(garecon, oracle, lambda: garecon.Engine(cluster_name="default"))
