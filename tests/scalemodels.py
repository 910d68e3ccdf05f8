"""Adversarial clusters at 10^4-10^5 objects: the generators of randmodel, multilbi, hotkeys and egbcases scaled up, so that
every row pass, index build, scan and compaction of a diff spans many blocks and tiles while the content still takes every
branch (bad hostnames, duplicate zones, load balancers and accelerators, orphans, wildcard records, broken annotations).

At these sizes randmodel's five zones are hot zones of about two records per object.  Its orphans are few whatever the size
(0-3), so `drop` removes a seeded fraction of the objects after generation: their accelerators, TXT owner values and alias
records stay in the AWS tables and become orphans of the full diff, and their keys are the deleted keys of gar_diff_keys."""
import random

import egbcases
import hotkeys
import multilbi
import randmodel

KIND = {"service": 0, "ingress": 1}
# deleted keys that match nothing: absent from the cache and from every owner value, and keys that are not "ns/name"
ABSENT_KEYS = [(0, "default/absent"), (1, "prod/never-existed"), (0, "no-slash"), (1, "a/b/c"), (1, "")]


def key_of(ob):
    return KIND[ob["kind"]], f'{ob["ns"]}/{ob["name"]}'


def drop(objects, seed, frac):
    """Remove a seeded `frac` of the objects.  -> (kept objects in their order, deleted keys of the dropped ones)."""
    rng = random.Random(seed * 104729 + 17)
    kept, gone = [], []
    for ob in objects:
        (gone if rng.random() < frac else kept).append(ob)
    return kept, [key_of(ob) for ob in gone]


def randmodel_dropped(seed, n_objects, frac=0.08):
    """randmodel at n_objects with `frac` of the objects dropped.  -> (objects, actual, deleted keys)."""
    objects, actual = randmodel.make(seed, n_objects=n_objects)
    kept, dropped = drop(objects, seed, frac)
    return kept, actual, dropped


def _interleave(rng, a, b):
    """The elements of a and b in one list, each list's own order kept, b's elements at random places."""
    at = sorted(rng.sample(range(len(a) + len(b)), len(b)))
    out, ia, ib = [], 0, 0
    for k in range(len(a) + len(b)):
        if ib < len(b) and at[ib] == k:
            out.append(b[ib])
            ib += 1
        else:
            out.append(a[ia])
            ia += 1
    return out


def hot_cluster(seed, n_objects, ndup_acc=140, ndup_alias=120, ndup_val=160):
    """hotkeys' duplicate chains (one owner with ndup_acc accelerators, one record name with ndup_alias alias records, TXT sets
    of ndup_val and 2 * ndup_val values) inside a randmodel cluster: the hot objects, accelerators and load balancers sit at
    random places of their lists, the hot records at the end of the cluster's example.com. zone."""
    rng = random.Random(seed * 7 + 3)
    objects, actual = randmodel.make(seed, n_objects=n_objects)
    hobj, hact = hotkeys.make(ndup_acc=ndup_acc, ndup_alias=ndup_alias, ndup_val=ndup_val)
    zone = next(z for z in actual["zones"] if z["name"] == "example.com.")
    zone["records"].extend(hact["zones"][0]["records"])
    actual["accelerators"] = _interleave(rng, actual["accelerators"], hact["accelerators"])
    actual["lbs"] = _interleave(rng, actual["lbs"], hact["lbs"])
    return _interleave(rng, objects, hobj), actual


def multilbi_cluster(seed, n_objects):
    return multilbi.make(seed, n_objects=n_objects)


def bindings_cluster(seed, n_objects, n_bindings, n_known=4000):
    """egbcases' random bindings over a randmodel cluster with thousands of known endpoint groups, one of them (known[0]) shared
    by a fifth of the bindings, and 2 % of the bindings with 64-191 endpoint ids.  -> (objects, actual, bindings, known)."""
    return egbcases.random_bindings(seed, n_objects=n_objects, n_bindings=n_bindings, n_known=n_known, hot=0.2, long=0.02)
