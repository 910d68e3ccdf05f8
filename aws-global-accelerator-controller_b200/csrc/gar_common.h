// gar_common.h — types and byte-level primitives shared by every kernel of the diff engine.
//
// All row logic is written as GAR_HD functions so that the very same code can be compiled (a) by nvcc into the
// sm_90a kernels that ship in libgarecon.so and (b) by g++ into tests/hostsim, a debugging build that lets
// the CPU-only CI run the device logic against the oracle.  (b) is a test artefact; the product has no CPU path.
#pragma once

#include <stdint.h>
#include <stddef.h>

#include "../../include/garecon.h"

#if defined(__CUDACC__)
#define GAR_HD __host__ __device__ __forceinline__
#define GAR_D __device__ __forceinline__
#else
#define GAR_HD inline
#define GAR_D inline
#endif

// Warp vote used to keep the outer loops of the decide kernels warp-uniform (and to force reconvergence at
// every iteration).  Only valid in kernels where all 32 lanes of every warp stay alive (for_each_warp).
#if defined(__CUDA_ARCH__)
#define GAR_ANY(p) __any_sync(0xffffffffu, (p))
#else
bool gar_host_vote(bool p);  // tests/hostsim: 32 host threads emulate a warp; a vote that not all lanes reach is an error
#define GAR_ANY(p) gar_host_vote((p))
#endif

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int32_t i32;
typedef int64_t i64;

#define GAR_SLAB_PAD 32  // bytes of readable zero padding the engine keeps after every slab (wide loads may over-read)

// ------------------------------------------------------------------ string views

struct Str {
  const u8 *p;
  u32 n;
};

GAR_HD Str mkstr(const u8 *slab, gar_str r) { return Str{slab + GAR_STR_OFF(r), GAR_STR_LEN(r)}; }
GAR_HD Str substr(Str s, u32 off, u32 n) { return Str{s.p + off, n}; }

// Unaligned little-endian 8-byte load built from two aligned ones.  May touch up to 15 bytes past p:
// every slab carries GAR_SLAB_PAD bytes of padding and slab bases are 16-byte aligned.
GAR_HD u64 ld64u(const u8 *p) {
  uintptr_t a = (uintptr_t)p;
  const u64 *q = (const u64 *)(a & ~(uintptr_t)7);
  unsigned sh = (unsigned)(a & 7) * 8;
  u64 lo = q[0], hi = q[1];
  return (lo >> sh) | ((hi << 1) << (63 - sh));  // branch-free: for sh == 0 the second term shifts out entirely
}
GAR_HD u64 lowmask(u32 nbytes) { return nbytes >= 8 ? ~0ull : ((1ull << (nbytes * 8)) - 1); }

// byte-exact equality, 8 bytes per step
GAR_HD bool streq(Str a, Str b) {
  if (a.n != b.n) return false;
  u32 i = 0;
  for (; i + 8 <= a.n; i += 8)
    if (ld64u(a.p + i) != ld64u(b.p + i)) return false;
  if (i < a.n) {
    u64 m = lowmask(a.n - i);
    if ((ld64u(a.p + i) & m) != (ld64u(b.p + i) & m)) return false;
  }
  return true;
}

// Comparisons with string literals: the literal is packed into 8-byte words at compile time (constant-folded), the
// string side is read 8 bytes per step; no byte loops.
GAR_HD constexpr u64 lit_word(const char *lit, u32 n, u32 i) {
  u64 w = 0;
  for (u32 k = 0; k < 8 && i + k < n; k++) w |= (u64)(u8)lit[i + k] << (8 * k);
  return w;
}
// a[off .. off+n) == lit, given off + n <= a.n
template <u32 N>
GAR_HD bool lit_eq_at(Str a, u32 off, const char (&lit)[N]) {
  constexpr u32 n = N - 1;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (u32 i = 0; i < n; i += 8) {
    u64 w = ld64u(a.p + off + i);
    if (n - i < 8) w &= lowmask(n - i);
    if (w != lit_word(lit, n, i)) return false;
  }
  return true;
}
#define STREQ_LIT(s, lit) ((s).n == (u32)(sizeof(lit) - 1) && lit_eq_at((s), 0, lit))
#define HAS_PREFIX_LIT(s, lit) ((s).n >= (u32)(sizeof(lit) - 1) && lit_eq_at((s), 0, lit))
#define HAS_SUFFIX_LIT(s, lit) ((s).n >= (u32)(sizeof(lit) - 1) && lit_eq_at((s), (s).n - (u32)(sizeof(lit) - 1), lit))

// ------------------------------------------------------------------ SWAR byte search (8 bytes per step)

GAR_HD u64 swar_eq_mask(u64 w, u8 c) {  // 0x80 in every byte of w that equals c (exact: no false positives below the first hit)
  u64 x = w ^ (0x0101010101010101ull * c);
  return (x - 0x0101010101010101ull) & ~x & 0x8080808080808080ull;
}
GAR_HD u32 ctz64(u64 x) {
#if defined(__CUDA_ARCH__)
  return (u32)(__ffsll((long long)x) - 1);
#else
  return (u32)__builtin_ctzll(x);
#endif
}
// index of the first byte == c in s[from..), or s.n
GAR_HD u32 find_byte(Str s, u32 from, u8 c) {
  for (u32 i = from; i < s.n; i += 8) {
    u64 m = swar_eq_mask(ld64u(s.p + i), c);
    if (s.n - i < 8) m &= lowmask(s.n - i);
    if (m) return i + (ctz64(m) >> 3);
  }
  return s.n;
}
// exact per-byte equality mask (0x80 in every byte of w equal to c; unlike swar_eq_mask, exact in every position)
GAR_HD u64 swar_eq_exact(u64 w, u8 c) {
  u64 x = w ^ (0x0101010101010101ull * c);
  return ~(((x & 0x7F7F7F7F7F7F7F7Full) + 0x7F7F7F7F7F7F7F7Full) | x) & 0x8080808080808080ull;
}
// 0x80 in every byte b of w with lo <= b <= hi; all bytes of w must be < 0x80 (caller checks), 0 < lo <= hi < 0x80
GAR_HD u64 swar_in_range(u64 w, u8 lo, u8 hi) {
  u64 ge = w + 0x0101010101010101ull * (u8)(0x80 - lo);
  u64 le = 0x0101010101010101ull * (u8)(0x80 | hi) - w;
  return ge & le & 0x8080808080808080ull;
}
GAR_HD u32 clz64(u64 x) {
#if defined(__CUDA_ARCH__)
  return (u32)__clzll((long long)x);
#else
  return (u32)__builtin_clzll(x);
#endif
}
GAR_HD u32 count_byte(Str s, u8 c) {  // byte-exact count (the SWAR mask can over-report bytes above the first hit, so count per byte)
  u32 n = 0;
  for (u32 i = find_byte(s, 0, c); i < s.n; i = find_byte(s, i + 1, c)) n++;
  return n;
}

// ------------------------------------------------------------------ xxHash64 (XXH64, seed 0) over contiguous bytes

#define XXP1 0x9E3779B185EBCA87ull
#define XXP2 0xC2B2AE3D27D4EB4Full
#define XXP3 0x165667B19E3779F9ull
#define XXP4 0x85EBCA77C2B2AE63ull
#define XXP5 0x27D4EB2F165667C5ull

GAR_HD u64 rotl64(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
GAR_HD u64 xx_round(u64 acc, u64 in) { return rotl64(acc + in * XXP2, 31) * XXP1; }
GAR_HD u64 xx_merge(u64 acc, u64 v) { return (acc ^ xx_round(0, v)) * XXP1 + XXP4; }
GAR_HD u64 xx_avalanche(u64 h) {
  h ^= h >> 33;
  h *= XXP2;
  h ^= h >> 29;
  h *= XXP3;
  h ^= h >> 32;
  return h;
}

// Key hash: xxHash64's round/avalanche applied to one 8-byte word per step (tail masked), so that the scalar
// form (index build, one thread per row) and the warp-uniform form (probes: all 32 lanes step together under a
// vote, gar_rows.h) walk a key in exactly the same number of equal steps.  Both sides of every join use it.
GAR_HD u64 hash_init(u32 n) { return XXP5 ^ ((u64)n * XXP3); }
GAR_HD u64 hash_word(u64 h, u64 w) { return rotl64(h ^ (w * XXP2), 31) * XXP1 + XXP4; }
GAR_HD u64 load_word(Str s, u32 i) {  // bytes [i, i+8) of s, zero beyond the end
  u64 w = ld64u(s.p + i);
  if (s.n - i < 8) w &= lowmask(s.n - i);
  return w;
}
GAR_HD u64 gar_hash(Str s) {
  u64 h = hash_init(s.n);
  for (u32 i = 0; i < s.n; i += 8) h = hash_word(h, load_word(s, i));
  return xx_avalanche(h);
}

// ---- warp-uniform string primitives: EVERY lane of the warp must call them (lanes without work pass act = false);
// each loop iteration is one GAR_ANY vote, so the lanes' loads issue together.
GAR_HD u64 u_hash(bool act, Str s) {
  u64 h = hash_init(s.n);
  const u32 n = act ? s.n : 0;
  for (u32 i = 0;; i += 8) {
    bool step = i < n;
    if (!GAR_ANY(step)) break;
    if (step) h = hash_word(h, load_word(s, i));
  }
  return xx_avalanche(h);
}
GAR_HD bool u_streq(bool act, Str a, Str b) {
  bool eq = act && a.n == b.n;
  const u32 n = eq ? a.n : 0;
  for (u32 i = 0;; i += 8) {
    bool step = eq && i < n;
    if (!GAR_ANY(step)) break;
    if (step) {
      u64 x = ld64u(a.p + i) ^ ld64u(b.p + i);  // one tail mask for both sides
      if (n - i < 8) x &= lowmask(n - i);
      if (x) eq = false;
    }
  }
  return eq;
}
GAR_HD u32 u_find_byte(bool act, Str s, u32 from, u8 c) {
  u32 found = s.n;
  bool done = !act;
  for (u32 i = from;; i += 8) {
    bool step = !done && i < s.n;
    if (!GAR_ANY(step)) break;
    if (!step) continue;
    u64 m = swar_eq_mask(ld64u(s.p + i), c);
    if (s.n - i < 8) m &= lowmask(s.n - i);
    if (m) {
      found = i + (ctz64(m) >> 3);
      done = true;
    }
  }
  return found;
}

// combine a small integer (kind, zone row ...) or a second hash into a key hash
GAR_HD u64 hmix(u64 a, u64 b) { return xx_avalanche(a * XXP1 + rotl64(b, 29) * XXP2 + XXP5); }

// ------------------------------------------------------------------ bucketed hash index (read side)
//
// An index is a CSR of buckets: bucket b owns entries [begin[b], begin[b+1]).  Entries of a bucket are
// sorted by build-side row, so walking a bucket yields matching rows in table order — which the change
// set's canonical order needs (duplicates are legal and ordered).  An entry is one 32-byte sector: the tag
// (upper half of the 64-bit key hash), the row, and a denormalised copy of what the probe needs next (string
// refs, parent rows, small enums), so a probe touches the entry and then the key bytes — no column chasing.
// A tag hit is always followed by a full key comparison by the caller: hash equality is never trusted.

struct alignas(32) IdxEntry {
  u32 tag, row, a0, a1;
  u64 s0, s1;
};

struct HashIdx {
  const u32 *begin;     // [nbuckets + 1]
  const IdxEntry *ent;  // [n_entries]
  u32 mask;             // nbuckets - 1 (nbuckets is a power of two)
};

struct Cursor {
  u32 pos, end, tag;
};

GAR_HD u32 hash_bucket(u64 h, u32 mask) { return (u32)h & mask; }
GAR_HD u32 hash_tag(u64 h) { return (u32)(h >> 32); }

GAR_HD IdxEntry load_entry(const IdxEntry *p) {
#if defined(__CUDA_ARCH__)
  const uint4 *q = reinterpret_cast<const uint4 *>(p);
  uint4 lo = __ldg(q), hi = __ldg(q + 1);
  IdxEntry e;
  e.tag = lo.x;
  e.row = lo.y;
  e.a0 = lo.z;
  e.a1 = lo.w;
  e.s0 = (u64)hi.x | ((u64)hi.y << 32);
  e.s1 = (u64)hi.z | ((u64)hi.w << 32);
  return e;
#else
  return *p;
#endif
}

GAR_HD Cursor idx_open(const HashIdx &ix, u64 h) {
  u32 b = hash_bucket(h, ix.mask);
  Cursor c;
  c.pos = ix.begin[b];
  c.end = ix.begin[b + 1];
  c.tag = hash_tag(h);
  return c;
}
// next entry whose tag matches; false when the bucket is exhausted
GAR_HD bool idx_next(const HashIdx &ix, Cursor &c, IdxEntry *out) {
  while (c.pos < c.end) {
    IdxEntry e = load_entry(ix.ent + c.pos++);
    if (e.tag == c.tag) {
      *out = e;
      return true;
    }
  }
  return false;
}
