"""Keys whose hashes collide in an index: a numpy mirror of the engine's key hashes and a birthday search for colliding pairs.

Every hash index of the engine (csrc/gar_common.h, "bucketed hash index") keeps the upper half of a 64-bit key hash as the
entry's tag and uses the low log2(nb) bits as the bucket; a tag hit is always followed by a full key compare.  A random test
almost never produces two different keys that agree on tag and bucket, so that compare would go untested.  find_pairs builds
such keys on purpose: distinct keys of equal length that agree on the tag and on the low `bits` bits, i.e. that share bucket
and tag in every index of at most 2**bits buckets.  The mirror is pinned bit for bit to the C++ functions by
test_hash_collisions.test_mirror_matches_the_device_hashes.
"""
import functools

import numpy as np

U64 = np.uint64
P1, P2, P3, P4, P5 = (U64(x) for x in (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5))
ALPHABET = b"0123456789abcdefghijklmnopqrstuvwxyz"

# ------------------------------------------------------------------ hash mirror (gar_common.h, gar_rows.h "key hashes")


def _rotl(x, r):
    return (x << U64(r)) | (x >> U64(64 - r))


def _avalanche(h):
    h = h ^ (h >> U64(33))
    h = h * P2
    h = h ^ (h >> U64(29))
    h = h * P3
    return h ^ (h >> U64(32))


def _as_u64(x):
    return np.asarray(x, dtype=np.uint64) if not isinstance(x, np.ndarray) else x.astype(np.uint64, copy=False)


def hash_matrix(mat: np.ndarray) -> np.ndarray:
    """gar_hash of every row of an (N, L) uint8 matrix (all keys L bytes long): one xxHash64 round per 8-byte little-endian
    word, the tail word zero-padded, the length folded into the seed."""
    n, length = mat.shape
    pad = (-length) % 8
    words = np.ascontiguousarray(np.pad(mat, ((0, 0), (0, pad)))).view("<u8")
    with np.errstate(over="ignore"):
        h = np.full(n, P5 ^ (U64(length) * P3), dtype=np.uint64)
        for w in range(words.shape[1]):
            h = _rotl(h ^ (words[:, w] * P2), 31) * P1 + P4
        return _avalanche(h)


def _bytes(s) -> bytes:
    return s if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8", "surrogatepass")


def gar_hash(s) -> int:
    b = _bytes(s)
    return int(hash_matrix(np.frombuffer(b, dtype=np.uint8).reshape(1, len(b)))[0])


def hmix(a, b):
    """hmix of gar_common.h on ints or uint64 arrays"""
    with np.errstate(over="ignore"):
        r = _avalanche(_as_u64(a) * P1 + _rotl(_as_u64(b), 29) * P2 + P5)
    return int(r) if np.ndim(r) == 0 else r


def key_hash_kinded(kind: int, nsname) -> int:
    return hmix(kind + 1, gar_hash(nsname))


def key_hash_lb(region, name) -> int:
    return hmix(gar_hash(region), gar_hash(name))


def key_hash_zoned_h(zone: int, name_hash):
    return hmix(zone + 0x100, name_hash)


def key_hash_zoned(zone: int, name) -> int:
    return key_hash_zoned_h(zone, gar_hash(name))


def key_hash_str(s) -> int:
    return gar_hash(s)


# vectorised forms for the search: (N, L) key matrix -> uint64 hashes (one function object per argument, so that find_pairs'
# cache recognises it)
@functools.lru_cache(maxsize=None)
def kinded_fn(kind):
    return lambda mat: hmix(kind + 1, hash_matrix(mat))


@functools.lru_cache(maxsize=None)
def lb_fn(region):
    hr = gar_hash(region)
    return lambda mat: hmix(hr, hash_matrix(mat))


@functools.lru_cache(maxsize=None)
def zoned_fn(zone):
    return lambda mat: hmix(zone + 0x100, hash_matrix(mat))


def tag(h: int) -> int:
    return h >> 32


def bucket(h: int, nb: int) -> int:
    return h & (nb - 1)


# ------------------------------------------------------------------ index sizing (gar_pipeline.h: arm_group_a, build_index, resolve_owners)

# rows per bucket: group A (ix_lb, ix_thost, ix_zone, ix_val, ix_alias, ix_obj), the deleted-key indexes (ix_owner, ix_val) and the
# binding index ix_eg go through build_index with these loads; ix_ovn is sized by the number of ALL values over 8
LOAD = dict(lb=1, owner=1, thost=1, zone=1, val=1, alias=2, obj=1, ovn=8, eg=1)


def next_pow2(x: int) -> int:
    p = 1
    while p < x:
        p <<= 1
    return p


def nbuckets(index: str, rows: int) -> int:
    """bucket count of `index` built over `rows` table rows (n_lbs, n_accels, n_zones, n_values, n_records, n_objects, n_values,
    n_known_egs): next_pow2(max(16, rows // load))"""
    r = rows // LOAD[index]
    return next_pow2(16 if r < 16 else r)


def table_rows(objects, actual, known_egs=()) -> dict:
    """rows each index is sized by, for a dict model of tables.pack"""
    actual = actual or {}
    zones = actual.get("zones", [])
    recs = [r for z in zones for r in z["records"]]
    nval = sum(len(r.get("values", [])) for r in recs)
    nacc = len(actual.get("accelerators", []))
    return dict(lb=len(actual.get("lbs", [])), owner=nacc, thost=nacc, zone=len(zones), val=nval, alias=len(recs), obj=len(objects),
                ovn=nval, eg=len(known_egs))


def assert_collide(h1: int, h2: int, index: str, rows: int, bits: int = 10):
    """precondition of a collision scenario: `index`, built over `rows` rows, has at most 2**bits buckets, and the two key hashes
    fall into the same bucket with the same tag (but are not equal: the keys themselves differ)"""
    nb = nbuckets(index, rows)
    assert nb <= 1 << bits, f"{index}: {rows} rows give {nb} buckets, more than the 2**{bits} the pair collides in"
    assert tag(h1) == tag(h2) and bucket(h1, nb) == bucket(h2, nb), f"{index}: {h1:#018x} and {h2:#018x} do not collide in {nb} buckets"


# ------------------------------------------------------------------ birthday search

ROUND = 1 << 22


def _candidates(prefix: bytes, free: int, suffix: bytes, start: int, count: int, mul: int, add: int) -> tuple[np.ndarray, np.ndarray]:
    """`count` distinct keys prefix + <free base-36 characters> + suffix: the counter i maps to (i * mul + add) mod 36**free,
    a bijection since mul is prime to 36"""
    space = 36 ** free
    i = np.arange(start, start + count, dtype=np.uint64)
    with np.errstate(over="ignore"):
        v = (i * U64(mul) + U64(add)) % U64(space)
    digits = np.empty((count, free), dtype=np.uint8)
    x = v.copy()
    alpha = np.frombuffer(ALPHABET, dtype=np.uint8)
    for k in range(free):
        digits[:, k] = alpha[(x % U64(36)).astype(np.intp)]
        x //= U64(36)
    mat = np.empty((count, len(prefix) + free + len(suffix)), dtype=np.uint8)
    mat[:, :len(prefix)] = np.frombuffer(prefix, dtype=np.uint8)
    mat[:, len(prefix):len(prefix) + free] = digits
    mat[:, len(prefix) + free:] = np.frombuffer(suffix, dtype=np.uint8)
    return mat, v


@functools.lru_cache(maxsize=None)
def _search(hash_fn, hash_fn_b, template: str, k: int, bits: int, seed: int, free: int):
    prefix, suffix = (s.encode() for s in template.split("{}"))
    space = 36 ** free
    mul = 1_000_003 + 2 * seed * 6  # prime to 36 (odd, not a multiple of 3)
    while mul % 3 == 0 or mul % 2 == 0:
        mul += 2
    add = (seed * 0x9E3779B97F4A7C15) % space
    sides = [hash_fn] if hash_fn_b is None else [hash_fn, hash_fn_b]
    keys, vals, side = [], [], []
    mask = (1 << bits) - 1
    start = 0
    while start + ROUND <= space:
        mat, v = _candidates(prefix, free, suffix, start, ROUND, mul, add)
        for s, fn in enumerate(sides):
            h = fn(mat)
            keys.append(((h >> U64(32)) << U64(bits)) | (h & U64(mask)))
            vals.append(v)
            side.append(np.full(ROUND, s, dtype=np.uint8))
        start += ROUND
        kk, vv, ss = np.concatenate(keys), np.concatenate(vals), np.concatenate(side)
        order = np.argsort(kk, kind="stable")
        kk, vv, ss = kk[order], vv[order], ss[order]
        hit = np.nonzero(kk[1:] == kk[:-1])[0]
        pairs, used = [], set()
        for j in hit:
            a, b = (j, j + 1) if ss[j] <= ss[j + 1] else (j + 1, j)
            if vv[a] == vv[b] or (hash_fn_b is not None and ss[a] == ss[b]) or vv[a] in used or vv[b] in used:
                continue
            used.update((vv[a], vv[b]))
            pairs.append((int(vv[a]), int(vv[b])))
            if len(pairs) == k:
                return tuple((_key(prefix, free, suffix, a), _key(prefix, free, suffix, b)) for a, b in pairs)
    raise AssertionError(f"no {k} colliding pairs for {template!r}")


def _key(prefix: bytes, free: int, suffix: bytes, v: int) -> str:
    d = bytearray()
    for _ in range(free):
        d.append(ALPHABET[v % 36])
        v //= 36
    return (prefix + bytes(d) + suffix).decode()


def find_pairs(hash_fn, template: str, k: int, bits: int = 10, seed: int = 0, hash_fn_b=None, free: int = 6) -> list[tuple[str, str]]:
    """k disjoint pairs (a, b) of distinct keys template.format(<free base-36 characters>): hash_fn(a) and hash_fn_b(b) (hash_fn
    when None) agree on the tag (upper 32 bits) and on the low `bits` bits.  Deterministic; candidates are searched in rounds of
    2**22 until k pairs turn up, and the result is cached for the session (the hash functions of kinded_fn, lb_fn and zoned_fn are
    one object per argument, and hash_matrix is gar_hash itself)."""
    return list(_search(hash_fn, hash_fn_b, template, k, bits, seed, free))


def differing_words(a: str, b: str) -> set:
    """the 8-byte words (index from 0) in which two equal-length keys differ"""
    x, y = _bytes(a), _bytes(b)
    assert len(x) == len(y)
    return {i // 8 for i in range(len(x)) if x[i] != y[i]}


# Templates that place the free bytes of a key (the only bytes in which the two keys of a pair differ) in
#   "first":  the first 8-byte word,
#   "middle": a middle word that is a full 8 bytes,
#   "tail":   the last word, which is shorter than 8 bytes (the key length is not a multiple of 8) and so compared under a mask.
# The object key templates are "ns/name"; the word each placement lands in is checked by placement_word().
OBJECT_KEYS = {"first": "{}/svc-collide", "middle": "default/{}-svc-x", "tail": "default/svc-col-{}"}
PLACEMENTS = sorted(OBJECT_KEYS)


def placement_word(template: str, placement: str, free: int = 6) -> int:
    """the word the free bytes of `template` occupy, checked against the placement's definition"""
    lo = template.index("{}")
    n = len(template) - 2 + free
    first, last = lo // 8, (lo + free - 1) // 8
    assert first == last, f"{template!r}: the free bytes straddle words {first} and {last}"
    if placement == "first":
        assert first == 0
    elif placement == "middle":
        assert 0 < first and (first + 1) * 8 <= n, f"{template!r}: not in a full word after the first"
    else:
        assert n % 8 != 0 and first == (n - 1) // 8, f"{template!r}: not in a masked tail word"
    return first


# One key whose Service hash and Ingress hash collide: key_hash_kinded(0, k) and key_hash_kinded(1, k) agree on the tag and on the
# low 7 bits.  Same-key pairs cannot come from a birthday search (each candidate is one 2**-39 trial), so this one was found
# once by an exhaustive multi-threaded walk over "default/k-" + 7 base-36 characters and is kept here; the mirror-pinning test
# re-checks the property against the C++ hash on every run.
SAME_KEY_BOTH_KINDS = "default/k-rurx7l3"
SAME_KEY_BITS = 7
