"""The rules of gar_read_set (include/garecon.h) restated in Python over the dict model, for tests/test_read_set.py.

It reads the reference's lists the way oracle/pyref.py does — pyref's own hostname tokeniser, zone walk (parent_domain), owner
tag names and annotation helpers — and answers each list call from maps built once per call, so that clusters of 10^4 objects
stay quick.  It is the arbiter for exact equality with the engine's read set."""
from oracle import pyref


def read_set(objects, actual, cluster, rows, deleted=()):
    """The resident AWS rows gar_read_set reports for a keyset (include/garecon.h), restated from the reference's lists:
    -> dict(lbs, accs, zones: sorted row lists, misses: [(object row, j, name, region)] sorted).  Rows are list positions (a
    model may repeat one dict at several positions)."""
    actual = actual or {}
    accs = list(enumerate(actual.get("accelerators", [])))
    lbs = list(enumerate(actual.get("lbs", [])))
    zones = list(enumerate(actual.get("zones", [])))
    lb_rows, acc_rows, zone_rows, misses = set(), set(), set(), set()
    # the reference's linear scans, answered from maps built once: first (region, name) row, accelerators by their effective
    # tags (a later duplicate tag wins, tags_contain), zone rows by dotted name (first wins), zones by record value
    first_lb, by_owner, by_host, zone_of_name, zones_of_value = {}, {}, {}, {}, {}
    for r, lb in lbs:
        first_lb.setdefault((lb["region"], lb["name"]), r)
    for r, a in accs:
        t = dict(a.get("tags", []))
        if t.get(pyref.TAG_MANAGED, "") == "true" and t.get(pyref.TAG_CLUSTER, "") == cluster:
            by_owner.setdefault(t.get(pyref.TAG_OWNER, ""), []).append(r)
            by_host.setdefault(t.get(pyref.TAG_HOST, ""), []).append(r)
    for r, z in zones:
        zone_of_name.setdefault(z["name"], r)
        for rec in z.get("records", []):
            for v in rec.get("values", []):
                zones_of_value.setdefault(v, set()).add(r)

    def hosted_zone(hostname):  # route53.go:335-358
        t = hostname
        while t != "":
            if t + "." in zone_of_name:
                return zone_of_name[t + "."]
            t = pyref.parent_domain(t)
        return None

    def owned(resource, key):  # ListGlobalAcceleratorByResource (:87-110) and the owner values of FindOwnered*RecordSets
        acc_rows.update(by_owner.get(f"{resource}/{key}", []))
        zone_rows.update(zones_of_value.get(f'"heritage=aws-global-accelerator-controller,cluster={cluster},{resource}/{key}"', ()))

    for i in rows:
        ob = objects[i]
        for j, h in enumerate(ob.get("lb_ingress", [])):
            code, name, region = pyref.tokenise(h)
            if code > 2:
                continue
            lb = first_lb.get((region, name))  # load_balancer.go:13-30: first row wins
            if lb is None:
                misses.add((i, j, name, region))
            else:
                lb_rows.add(lb)
            acc_rows.update(by_host.get(h, [])[:2])  # ListGlobalAcceleratorByHostname (:62-85): the count gate reads two
        owned(pyref._resource(ob), f"{ob.get('ns', 'default')}/{ob['name']}")
        ann = pyref._ann(ob)
        if pyref.ANN_R53 in ann:
            for piece in ann[pyref.ANN_R53].split(","):
                z = hosted_zone(piece)
                if z is not None:
                    zone_rows.add(z)
    for kind, key in deleted:
        owned("service" if kind == 0 else "ingress", key)
    return {"lbs": sorted(lb_rows), "accs": sorted(acc_rows), "zones": sorted(zone_rows), "misses": sorted(misses)}
