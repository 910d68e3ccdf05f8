"""EndpointGroupBinding cases (pkg/controller/endpointgroupbinding/reconcile.go): one hand-written case per branch of
reconcileDelete / reconcileCreate / reconcileUpdate, and a seeded random model on top of randmodel's snapshot."""
import importlib
import random

import randmodel

pyref = importlib.import_module("oracle.pyref")

EG = "arn:aws:globalaccelerator::1:accelerator/a/listener/l/endpoint-group/"


def _lb(i, region="us-west-2", state="active"):
    name = f"lb{i:03d}"
    return dict(region=region, name=name, dns=f"{name}-0123456789abcdef.elb.{region}.amazonaws.com", arn=f"arn:aws:elasticloadbalancing:{region}:1:loadbalancer/net/{name}/{i:016x}",
                state=state)


def hand_cases():
    """Returns (objects, actual, bindings, known_egs); tests/test_bindings.py holds the hand-derived expectations by index."""
    lbs = [_lb(0), _lb(1), _lb(2), _lb(3, state="provisioning"), _lb(4, region="eu-west-1"), _lb(5)]
    svc = lambda name, hosts: dict(kind="service", ns="default", name=name, spec_type="LoadBalancer", annotations={}, lb_ingress=hosts, ports=[(80, "TCP")])
    objects = [
        svc("one", [lbs[0]["dns"]]),
        svc("two", [lbs[0]["dns"], lbs[1]["dns"]]),
        svc("dup", [lbs[1]["dns"], lbs[1]["dns"], lbs[2]["dns"]]),
        svc("none", []),
        svc("notelb", ["example.com"]),
        svc("unknown", ["lb999-0123456789abcdef.elb.us-west-2.amazonaws.com"]),
        svc("prov", [lbs[3]["dns"]]),
        svc("tworegions", [lbs[0]["dns"], lbs[4]["dns"]]),
        svc("tworegions-rev", [lbs[4]["dns"], lbs[0]["dns"]]),
        # the ALB form <name>-<id>.<region>.elb.amazonaws.com: the name is everything before the last "-<id>" of the first label
        dict(kind="ingress", ns="default", name="one", ingress_class="alb", annotations={}, lb_ingress=["k8s-alb5-0123456789.us-west-2.elb.amazonaws.com"], ports=[80]),
        dict(kind="ingress", ns="other", name="ing", ingress_class="alb", annotations={}, lb_ingress=[lbs[2]["dns"]], ports=[80]),
    ]
    lbs.append(dict(region="us-west-2", name="k8s-alb5", dns="k8s-alb5-0123456789.us-west-2.elb.amazonaws.com", arn="arn:alb5", state="active"))
    arn = lambda i: lbs[i]["arn"]
    known = [EG + "ok", EG + "ok2"]
    B = lambda **kw: dict(dict(ns="default", ref=("service", "one"), eg_arn=EG + "ok", deleting=False, finalizers=True, observed=True, endpoint_ids=[]), **kw)
    bindings = [
        # reconcileDelete
        B(deleting=True),                                                   # no endpoints: remove finalizer
        B(deleting=True, endpoint_ids=[arn(0)], eg_arn=EG + "gone"),        # EG not found: remove finalizer
        B(deleting=True, endpoint_ids=[arn(0)]),                            # n=1
        B(deleting=True, endpoint_ids=[arn(0), arn(1)]),                    # n=2: aliasing bug, panic on i=1
        B(deleting=True, endpoint_ids=[arn(0), arn(1), arn(2)]),            # n=3
        B(deleting=True, endpoint_ids=[arn(0), arn(1), arn(2), arn(5), arn(4)]),
        B(deleting=True, finalizers=False),
        # reconcileCreate
        B(finalizers=False),
        B(finalizers=False, ref=("service", "missing")),
        # reconcileUpdate
        B(endpoint_ids=[arn(0)]),                                           # in sync
        B(endpoint_ids=[arn(0)], observed=False),                           # in sync but new generation: weights + status
        B(),                                                                # add one
        B(ref=("service", "two")),                                          # add two
        B(ref=("service", "two"), endpoint_ids=[arn(1)]),                   # add the first only
        B(ref=("service", "two"), endpoint_ids=[arn(2), arn(1), arn(5)]),   # remove two, add one
        B(ref=("service", "dup"), endpoint_ids=[]),                         # duplicate hostnames: one arn once
        B(ref=("service", "dup"), endpoint_ids=[arn(0), arn(0)]),           # duplicate status ids: removed twice
        B(ref=("service", "none"), endpoint_ids=[]),                        # no hostnames, nothing to do
        B(ref=("service", "none"), endpoint_ids=[], observed=False),        # no hostnames, status only
        B(ref=("service", "none"), endpoint_ids=[arn(0)]),                  # nil regional client
        B(ref=None, endpoint_ids=[arn(0)]),                                 # neither ref: same nil client
        B(ref=None),
        B(ref=("service", "missing")),                                      # lister NotFound
        B(ref=("ingress", "two")),                                          # kind matters
        B(ref=("ingress", "one")),                                          # ALB hostname
        B(ns="other", ref=("ingress", "ing")),                              # namespace of the binding
        B(ns="other", ref=("service", "one")),
        B(ref=("service", "notelb")),
        B(ref=("service", "unknown")),
        B(ref=("service", "prov")),                                         # LB not active: requeue 30s
        B(ref=("service", "prov"), endpoint_ids=[arn(0)]),                  # remove happens before the requeue
        B(ref=("service", "one"), eg_arn=EG + "gone"),                      # DescribeEndpointGroup fails
        B(ref=("service", "one"), eg_arn=EG + "gone", endpoint_ids=[arn(0)]),  # in sync: never describes
        B(ref=("service", "tworegions")),                                   # add looks lb000 up in eu-west-1: not found
        B(ref=("service", "tworegions-rev")),                               # add looks lb004 up in us-west-2: not found
        B(ref=("service", "tworegions"), endpoint_ids=[arn(0)]),            # only the last one is new: found
        B(ref=("service", "one"), eg_arn=EG + "ok2", endpoint_ids=[arn(1)]),
    ]
    return objects, dict(lbs=lbs), bindings, known


def random_bindings(seed: int, n_objects: int = 40, n_bindings: int = 120, n_known: int = 6, hot: float = 0.0, long: float = 0.0):
    """n_known endpoint groups, all but the last known to AWS; a fraction `hot` of the bindings all name the first one and a
    fraction `long` carry 64-191 extra endpoint ids.  Those two draw from a second generator, so that with hot = long = 0 the
    model is the same as without them."""
    rng = random.Random(seed * 7919 + 13)
    extra = random.Random(seed * 7919 + 14)
    objects, actual = randmodel.make(seed, n_objects=n_objects)
    lbs = actual.get("lbs", [])
    arns = [lb["arn"] for lb in lbs] + ["arn:stale:1", "arn:stale:2"]
    first_arn = {}  # (name, region) -> ARN of the first load balancer of that name in that region
    for lb in lbs:
        first_arn.setdefault((lb["name"], lb["region"]), lb["arn"])
    known = [EG + str(i) for i in range(n_known)]
    bindings = []
    for _ in range(n_bindings):
        ob = rng.choice(objects) if objects and rng.random() < 0.9 else None
        if ob is None:
            ref = None if rng.random() < 0.5 else (rng.choice(["service", "ingress"]), "nope")
            ns = "default"
        else:
            kind = ob.get("kind", "service") if rng.random() < 0.95 else rng.choice(["service", "ingress"])
            ref, ns = (kind, ob["name"]), ob.get("ns", "default")
        ids = []
        r = rng.random()
        if ob is not None and r < 0.6 and lbs:
            # start from the object's own load balancers, then perturb
            for h in ob.get("lb_ingress", []):
                t = pyref.tokenise(h)
                if t[0] < 3 and (t[1], t[2]) in first_arn:
                    ids.append(first_arn[t[1], t[2]])
            if rng.random() < 0.4 and ids:
                ids.pop(rng.randrange(len(ids)))
            if rng.random() < 0.3:
                ids.insert(rng.randrange(len(ids) + 1), rng.choice(arns))
        elif r < 0.85:
            ids = [rng.choice(arns) for _ in range(rng.randrange(0, 5))]
        b = dict(ns=ns, ref=ref, eg_arn=rng.choice(known + [EG + "gone"]), deleting=rng.random() < 0.2, finalizers=rng.random() < 0.85,
                 observed=rng.random() < 0.7, endpoint_ids=ids)
        if hot and extra.random() < hot:
            b["eg_arn"] = known[0]
        if long and extra.random() < long:
            b["endpoint_ids"] = ids + [extra.choice(arns) for _ in range(extra.randrange(64, 192))]
        bindings.append(b)
    return objects, actual, bindings, known[:-1]
