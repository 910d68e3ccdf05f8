// gar_pipeline.h — the diff as a sequence of data-parallel stages over a Backend.
//
// Backend = how a stage runs: the CUDA backend (gar_engine.cu) launches sm_90a kernels on a stream; the
// host-simulation backend (tests/hostsim) runs the same functors in loops so the CPU-only test tier can
// exercise the device logic.  Stages, functors and their order live here once.
//
// Backend interface:
//   template <class F> void for_each(const char *name, u32 n, const F &f);  // f(i) for i in [0, n)
//   template <class F> void for_each_warp(const char *name, u32 n, const F &f);  // f(i, i < n) for i in [0, roundup(n, 32)):
//                                                                                // full warps, f may use GAR_ANY votes
//   void exclusive_scan(u32 *data, u32 n);                                  // in place
//   void sort_pairs(u32 *keys, u32 *vals, u32 *keys_alt, u32 *vals_alt, u32 n, int bits);  // stable, result in keys/vals
//   void fill32(u32 *p, u32 value, size_t n);
//   void *ensure(int slot, size_t bytes);                                   // scratch buffer `slot`, at least `bytes`
//   template <class F> void for_each_staged(const char *name, u32 n, const F &f);  // f(i), or f.run(i, view) with string windows staged on chip
//   template <class... Fs> void for_each_multi(const char *name, std::initializer_list<u32> ns, const Fs &...fs);  // ONE launch: fs[k](i), i < ns[k]
//   template <class F> void for_each_dyn(const char *name, const u32 *n_dev, u32 cap, const F &f);       // f(i) for i < min(*n_dev, cap); the count
//   template <class F> void for_each_warp_dyn(const char *name, const u32 *n_dev, u32 cap, const F &f);  //   lives on the device: no read-back
//   void download(void *host_dst, const void *dev_src, size_t bytes);       // blocking
//   int graph_begin(u64 signature);  void graph_end();                      // launch-sequence caching (CUDA graphs): 0 = run the
//                                                                           // launches, 1 = run them while they are recorded, 2 = replayed
//   void download_start(int id, const void *dev_src, size_t bytes);         // id 0..1: small read-back in flight while later
//   void download_wait(int id, void *host_dst, size_t bytes);               //   stages are queued; wait blocks only if needed
#pragma once

#include <stdio.h>
#include <stdlib.h>

#include <initializer_list>

#include "gar_rows.h"

#if defined(__CUDA_ARCH__)
#define GAR_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#else
#define GAR_ATOMIC_ADD(p, v) (*(p) += (v))
#endif

// ------------------------------------------------------------------ scratch slots

enum Slot {
  S_DERIVED, S_OFLAGS, S_OKEY_HASH, S_STAGE_GA, S_STAGE_R53, S_ANN_R53, S_ANN_NAME, S_ANN_TAGS, S_ANN_LISTEN, S_DPORT_BEGIN, S_DPORTS,
  S_TOK_CODE, S_TOK_NAME, S_TOK_REGION,
  S_ACC_FLAGS, S_ACC_OWNER_KEY, S_ACC_OWNER, S_ACC_THOST, S_ACC_MANAGED, S_ACC_OWNER_HASH, S_ACC_THOST_HASH, S_REC_NAME_HASH, S_VAL_KEY_HASH,
  S_REC_ZONE, S_VAL_REC, S_VAL_CLS, S_VAL_KEY, S_VAL_ORPHAN, S_VAL_LINK, S_ACC_DIGEST,
  S_R53_MODE, S_R53_ACC, S_R53_ACC_DNS, S_PAIR_BEGIN, S_PAIR_OBJ, S_PAIR_HN, S_PAIR_CODE, S_PAIR_ZONE, S_PAIR_REC,
  S_IX_LB, S_IX_OWNER = S_IX_LB + 3, S_IX_THOST = S_IX_OWNER + 3, S_IX_ZONE = S_IX_THOST + 3, S_IX_VAL = S_IX_ZONE + 3,
  S_IX_ALIAS = S_IX_VAL + 3, S_IX_OBJ = S_IX_ALIAS + 3, S_IX_OVN = S_IX_OBJ + 3,
  S_SORT_KEYS = S_IX_OVN + 3, S_SORT_VALS, S_SORT_KEYS_ALT, S_SORT_VALS_ALT, S_SORT_TAGS,
  S_COUNTS, S_STATUS_GA, S_STATUS_R53, S_OPS, S_ERRFLAG, S_IX_EG, S_IX_EG_ENT, S_IX_EG_PAD,
  S_VAL_OBJ, S_ACC_OBJ, S_OBJ_CANON, S_OWN_BEGIN, S_OWN_FILL, S_OWN_ENT, S_OWN_MULTI,
  S_IXA_BEGIN, S_IXA_FILL, S_IXA_ENT, S_IXA_MULTI, S_OVN_FILL, S_OVN_MULTI, S_LB_HASH, S_REC_FLAGS, S_LBI_RES,
  S_NSLOTS
};

// ------------------------------------------------------------------ functors (one per stage)

struct FClassify {
  DevTables T;
  Work W;
  u32 *derived_public;
  u8 *oflags;
  u32 *errflag;
  GAR_HD void operator()(u32 i) const {
    classify_object(T, W, i);
    W.obj_canon[i] = i;  // rows that repeat an earlier row's key are redirected when ix_obj is ordered (canon_bucket)
    u32 dv = W.derived[i];
    if (dv & OBJ_KEY_BAD) GAR_ATOMIC_ADD(errflag, 1u);
    derived_public[i] = dv & 0xFFu;
  }
};
// "Staged" row passes (CUDA backend: gar_engine.cu k_for_each_staged): with column-major slabs the strings of one column of a
// block's consecutive rows are ONE contiguous byte range, so the block fetches that range with a single TMA bulk copy
// (cp.async.bulk + mbarrier) into shared memory and parses from there.  A functor describes up to 2 windows:
//   stage_window(c, r0, r1, &lo, &hi)  slab byte range [lo, hi) that holds column c's strings of rows [r0, r1)  (false: none)
//   stage_slab(c)                      the slab the window lives in
//   run(i, view)                       the row logic; view(c, ref) yields the string from shared memory when it lies inside the
//                                      staged window and from the slab otherwise (other layouts simply fall back per string)
struct FTokenise {
  DevTables T;
  Work W;
  static constexpr int kStageCols = 1;
  static constexpr u32 kStageBytes = 24 * 1024;  // 256 lbIngress hostnames of ~70 bytes
  static constexpr bool kStageByDefault = true;  // H100 SXM: 0.146 ms staged vs 0.149 ms direct
  GAR_HD void operator()(u32 i) const { tokenise_hostname(T, W, i); }
  GAR_HD const u8 *stage_slab(int) const { return T.o.slab; }
  GAR_HD bool stage_window(int, u32 r0, u32 r1, u64 *lo, u64 *hi) const {
    gar_str a = T.o.lbi_hostname[r0], b = T.o.lbi_hostname[r1 - 1];
    *lo = GAR_STR_OFF(a);
    *hi = GAR_STR_OFF(b) + GAR_STR_LEN(b);
    return true;
  }
  template <class View>
  GAR_HD void run(u32 i, const View &view) const { tokenise_hostname_at(T, W, i, view(0, T.o.lbi_hostname[i])); }
};
struct FDigestAccel {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 i) const { digest_accelerator(T, W, i); }
};
// child row -> parent row for a CSR (binary search on the begin array)
struct FExpand {
  const u32 *begin;
  u32 nparents;
  u32 *parent_of;
  GAR_HD void operator()(u32 c) const {
    u32 lo = 0, hi = nparents;  // last p with begin[p] <= c
    while (hi - lo > 1) {
      u32 mid = (lo + hi) >> 1;
      if (begin[mid] <= c) lo = mid;
      else hi = mid;
    }
    parent_of[c] = lo;
  }
};
// record row -> zone row, the hash of the record name (every (zone, name) key is derived from it), and its values: value ->
// record, owner-value classification.  One pass over the record table: a record's name and values are neighbours in the slab,
// so they share DRAM sectors.  A record set with MANY values (one hot TXT name claimed by thousands of owners) is not walked
// by its one thread: it goes on a list that FClassifyBigRecords works through with whole blocks.
constexpr u32 REC_INLINE_VALUES = 32;   // more values than this: a whole block works on the record
constexpr u32 REC_HUGE_VALUES = 4096;   // more than this: the whole grid does
struct DirectView {  // the un-staged view: every string comes from its slab
  const u8 *slab;
  GAR_HD Str operator()(int, gar_str r) const { return mkstr(slab, r); }
};
struct FPrepareRecord {
  DevTables T;
  Work W;
  u32 *big, *huge;  // [0] = count, then record rows
  static constexpr int kStageCols = 2;  // window 0: record names, window 1: the records' values
  static constexpr u32 kStageBytes = 16 * 1024;  // 256 names of ~28 bytes; ~130 values of ~95 bytes
  static constexpr bool kStageByDefault = true;  // H100 SXM: 0.418 ms staged vs 0.430 ms direct (bench.py, 10^6 objects)
  GAR_HD const u8 *stage_slab(int) const { return T.a.slab; }
  GAR_HD bool stage_window(int c, u32 r0, u32 r1, u64 *lo, u64 *hi) const {
    if (c == 0) {
      gar_str a = T.a.rec_name[r0], b = T.a.rec_name[r1 - 1];
      *lo = GAR_STR_OFF(a);
      *hi = GAR_STR_OFF(b) + GAR_STR_LEN(b);
      return true;
    }
    u32 v0 = T.a.rec_val_begin[r0], v1 = T.a.rec_val_begin[r1];
    if (v1 == v0) return false;
    gar_str a = T.a.val_value[v0], b = T.a.val_value[v1 - 1];
    *lo = GAR_STR_OFF(a);
    *hi = GAR_STR_OFF(b) + GAR_STR_LEN(b);
    return true;
  }
  GAR_HD void operator()(u32 r) const { run(r, DirectView{T.a.slab}); }
  template <class View>
  GAR_HD void run(u32 r, const View &view) const {
    u32 lo = 0, hi = T.a.n_zones;
    while (hi - lo > 1) {
      u32 mid = (lo + hi) >> 1;
      if (T.a.zone_rec_begin[mid] <= r) lo = mid;
      else hi = mid;
    }
    W.rec_zone[r] = lo;
    const Str nm = view(0, T.a.rec_name[r]);
    const u64 nh = gar_hash(nm);
    W.rec_name_hash[r] = nh;
    W.rec_flags[r] = find_byte(nm, 0, '\\') < nm.n ? 1 : 0;
    if (T.a.rec_has_alias[r]) ix_count(W.hist[IX_ALIAS], key_hash_zoned_h(lo, nh));
    u32 v0 = T.a.rec_val_begin[r], v1 = T.a.rec_val_begin[r + 1];
    if (v1 - v0 > REC_INLINE_VALUES) {
      u32 *list = v1 - v0 > REC_HUGE_VALUES ? huge : big;
#if defined(__CUDA_ARCH__)
      list[1 + atomicAdd(list, 1u)] = r;
#else
      list[1 + list[0]++] = r;
#endif
      return;
    }
    for (u32 v = v0; v < v1; v++) {
      W.val_rec[v] = r;
      classify_value_at(T, W, v, view(1, T.a.val_value[v]));
    }
  }
};
// fixed grid of BIG_BLOCKS x 256 threads: block b takes big records b, b + BIG_BLOCKS, ... and its threads stride over the
// values; the (few) huge records are strided over by the whole grid
constexpr u32 BIG_BLOCKS = 528;  // 4 x 132 SMs (H100 SXM)
struct FClassifyBigRecords {
  DevTables T;
  Work W;
  const u32 *big, *huge;
  GAR_HD void operator()(u32 i) const {
    const u32 blk = i >> 8, tid = i & 255u, nbig = big[0], nhuge = huge[0];
    for (u32 k = blk; k < nbig; k += BIG_BLOCKS) {
      u32 r = big[1 + k];
      for (u32 v = T.a.rec_val_begin[r] + tid; v < T.a.rec_val_begin[r + 1]; v += 256) {
        W.val_rec[v] = r;
        classify_value(T, W, v);
      }
    }
    for (u32 k = 0; k < nhuge; k++) {
      u32 r = huge[1 + k];
      for (u32 v = T.a.rec_val_begin[r] + i; v < T.a.rec_val_begin[r + 1]; v += BIG_BLOCKS * 256) {
        W.val_rec[v] = r;
        classify_value(T, W, v);
      }
    }
  }
};
struct FJsonCount {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 i) const {
    u32 n = 0;
    if (W.derived[i] & GAR_DV_PORTS_FROM_ANN) {
      u32 stk[GAR_JSON_STACK_WORDS];
      int c = json_listen_ports(mkstr(T.o.slab, W.ann_listen[i]), nullptr, stk);
      n = c < 0 ? 0u : (u32)c;
    }
    W.dport_begin[i] = n;
  }
};
struct FJsonWrite {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 i) const {
    if (!(W.derived[i] & GAR_DV_PORTS_FROM_ANN)) return;
    if (W.dport_begin[i + 1] == W.dport_begin[i] || W.dport_begin[i + 1] > W.dport_cap) return;
    u32 stk[GAR_JSON_STACK_WORDS];
    json_listen_ports(mkstr(T.o.slab, W.ann_listen[i]), W.dports + W.dport_begin[i], stk);
  }
};

// --- index rows: one functor per index says whether a row is indexed, its key hash and its entry payload
// (payload conventions: gar_rows.h "index probes").  The key pass streams the table once (coalesced) and leaves a
// complete 32-byte entry per row; the build then only moves entries.
// (region, name) hash of every load balancer: the only index key that is not produced by a row-local pass anyway
struct FLbHash {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 i) const {
    u64 h = key_hash_lb(mkstr(T.a.slab, T.a.lb_region[i]), mkstr(T.a.slab, T.a.lb_name[i]));
    W.lb_hash[i] = h;
    ix_count(W.hist[IX_LB], h);
  }
};
struct FRowLb {
  DevTables T;
  Work W;
  GAR_HD bool make(u32 i, u64 *h, IdxEntry *e) const {
    *h = W.lb_hash[i];
    e->a0 = T.a.lb_state[i];
    e->a1 = 0;
    e->s0 = T.a.lb_name[i];
    e->s1 = T.a.lb_region[i];
    return true;
  }
};
struct FRowOwner {
  DevTables T;
  Work W;
  GAR_HD bool make(u32 i, u64 *h, IdxEntry *e) const {
    u32 fl = W.acc_flags[i];
    *h = W.acc_owner_hash[i];
    e->a0 = fl;
    e->a1 = 0;
    e->s0 = W.acc_owner_key[i];
    e->s1 = 0;
    return (fl & ACC_MINE) && (fl & ACC_OWNER_KEYED) && i < W.acc_guest_from;
  }
};
struct FRowThost {
  DevTables T;
  Work W;
  GAR_HD bool make(u32 i, u64 *h, IdxEntry *e) const {
    *h = W.acc_thost_hash[i];
    e->a0 = e->a1 = 0;
    e->s0 = W.acc_thost[i];
    e->s1 = T.a.acc_dns[i];
    return (W.acc_flags[i] & ACC_MINE) != 0 && (!W.sharded || i >= W.acc_guest_from);
  }
};
struct FRowZone {
  DevTables T;
  GAR_HD bool make(u32 i, u64 *h, IdxEntry *e) const {
    Str zn = mkstr(T.a.slab, T.a.zone_name[i]);
    bool valid = zn.n >= 1 && zn.p[zn.n - 1] == '.';
    *h = valid ? key_hash_str(substr(zn, 0, zn.n - 1)) : 0;
    e->a0 = e->a1 = 0;
    e->s0 = T.a.zone_name[i];
    e->s1 = 0;
    return valid;
  }
};
struct FZoneLenMask {
  DevTables T;
  Work W;
  unsigned long long *mask;  // [4]
  GAR_HD void operator()(u32 z) const {
    Str zn = mkstr(T.a.slab, T.a.zone_name[z]);
    if (zn.n < 1 || zn.p[zn.n - 1] != '.') return;  // not indexed (FRowZone)
    ix_count(W.hist[IX_ZONE], key_hash_str(substr(zn, 0, zn.n - 1)));
    u32 b = zn.n - 1 < 255 ? zn.n - 1 : 255;
#if defined(__CUDA_ARCH__)
    atomicOr(&mask[b >> 6], 1ull << (b & 63));
#else
    mask[b >> 6] |= 1ull << (b & 63);
#endif
  }
};
struct FRowVal {
  DevTables T;
  Work W;
  GAR_HD bool make(u32 v, u64 *h, IdxEntry *e) const {
    u32 cls = W.val_cls[v];
    *h = W.val_key_hash[v];
    if (cls == VAL_NOT_OWNER) return false;
    u32 rec = W.val_rec[v];
    u32 kind = (cls & VAL_OWNER_INGRESS) ? 1u : 0u;
    u32 bs = (W.rec_flags[rec] & 1) ? VALNAME_HAS_BACKSLASH : 0u;
    e->a0 = rec;
    e->a1 = W.rec_zone[rec] | bs | (kind << 31);
    e->s0 = W.val_key[v];
    e->s1 = T.a.rec_name[rec];
    return true;
  }
};
struct FRowAlias {
  DevTables T;
  Work W;
  GAR_HD bool make(u32 r, u64 *h, IdxEntry *e) const {
    *h = key_hash_zoned_h(W.rec_zone[r], W.rec_name_hash[r]);
    e->a0 = W.rec_zone[r];
    e->a1 = T.a.rec_type[r];
    e->s0 = T.a.rec_name[r];
    e->s1 = T.a.rec_alias_dns[r];
    return T.a.rec_has_alias[r] != 0;
  }
};
struct FRowObj {
  DevTables T;
  Work W;
  GAR_HD bool make(u32 i, u64 *h, IdxEntry *e) const {
    gar_str ns = T.o.obj_ns[i];
    *h = W.okey_hash[i];
    e->a0 = T.o.obj_kind[i];
    e->a1 = 0;
    e->s0 = GAR_STR(GAR_STR_OFF(ns), GAR_STR_LEN(ns) + 1 + GAR_STR_LEN(T.o.obj_name[i]));
    e->s1 = 0;
    return !(W.derived[i] & OBJ_KEY_BAD);
  }
};
struct FRowOvn {
  DevTables T;
  Work W;
  GAR_HD bool make(u32 v, u64 *h, IdxEntry *e) const {
    u32 rec = W.val_rec[v];
    *h = key_hash_zoned_h(W.rec_zone[rec], W.rec_name_hash[rec]);
    e->a0 = rec;
    e->a1 = W.rec_zone[rec];
    e->s0 = T.a.rec_name[rec];
    e->s1 = T.a.val_value[v];
    return W.val_orphan[v] != 0;
  }
};

// Index build.  Fast path: (1) idx_rows: per row, entry + bucket key + bucket histogram; (2) scan; (3) idx_place: every
// indexed row drops its entry into its bucket with an atomic cursor (any order); (4) idx_order: buckets with >= 2
// entries are sorted by row id, which makes the result identical to a stable sort.  Buckets larger than
// IDX_SMALL_BUCKET (a hot key / adversarial input) raise `overflow`; the pipeline then rebuilds with the stable
// radix sort (idx_gather).
constexpr u32 IDX_SMALL_BUCKET = 48;
// ix_obj only: the ordering pass also writes the duplicate-key exceptions of Work::obj_canon (buckets [b0, b1) of the begin
// array it orders are ix_obj buckets; canon == nullptr: none)
struct CanonHook {
  u32 *canon;
  const u8 *slab;
  u32 b0, b1;
  GAR_HD void operator()(u32 b, const IdxEntry *ent, u32 lo, u32 m) const {
    if (canon && b >= b0 && b < b1) canon_bucket(ent, lo, m, slab, canon);
  }
};
template <class RowF>
struct FIdxRows {
  RowF rowf;
  u32 *keys, *vals;
  IdxEntry *tmp;
  u32 *counts;
  u32 mask, nb;
  GAR_HD void operator()(u32 i) const {
    u64 h = 0;
    IdxEntry e;
    bool valid = rowf.make(i, &h, &e);
    u32 k = valid ? hash_bucket(h, mask) : nb;  // rows that are not indexed carry the sentinel key nb
    keys[i] = k;
    if (vals) vals[i] = i;  // only the radix rebuild sorts (key, row) pairs
    if (valid) {
      e.tag = hash_tag(h);
      e.row = i;
      tmp[i] = e;
      GAR_ATOMIC_ADD(&counts[k], 1u);
    }
  }
};
struct FIdxPlace {
  const u32 *keys;
  u32 *cursor;  // [nb] starts as a copy of begin[]
  const IdxEntry *tmp;
  IdxEntry *ent;
  u32 nb;
  GAR_HD void operator()(u32 i) const {
    u32 k = keys[i];
    if (k == nb) return;
#if defined(__CUDA_ARCH__)
    u32 pos = atomicAdd(&cursor[k], 1u);
#else
    u32 pos = cursor[k]++;
#endif
    ent[pos] = tmp[i];
  }
};
struct FIdxOrder {
  const u32 *begin;
  IdxEntry *ent;
  u32 *overflow;
  CanonHook canon;
  GAR_HD void operator()(u32 b) const {
    u32 lo = begin[b], m = begin[b + 1] - lo;
    if (m < 2) return;
    if (m > IDX_SMALL_BUCKET) {
      GAR_ATOMIC_ADD(overflow, 1u);
      return;
    }
    for (u32 k = 1; k < m; k++) {  // insertion sort of 32-byte entries by row id, in place
      IdxEntry x = ent[lo + k];
      u32 j = k;
      while (j > 0 && ent[lo + j - 1].row > x.row) {
        ent[lo + j] = ent[lo + j - 1];
        j--;
      }
      if (j != k) ent[lo + j] = x;
    }
    canon(b, ent, lo, m);
  }
};
struct FIdxGather {  // radix fallback: position p of the stable sorted order holds row vals[p]
  const u32 *vals;
  const u32 *nvalid;
  const IdxEntry *tmp;
  IdxEntry *ent;
  GAR_HD void operator()(u32 p) const {
    if (p < *nvalid) ent[p] = tmp[vals[p]];
  }
};
struct FIdxCanon {  // radix fallback of ix_obj: the duplicate-key pass over the (already ordered) buckets
  const u32 *begin;
  const IdxEntry *ent;
  CanonHook canon;
  GAR_HD void operator()(u32 b) const {
    const u32 lo = begin[b], m = begin[b + 1] - lo;
    if (m >= 2) canon(b, ent, lo, m);
  }
};
// One-pass build (the default): the row-local passes have already counted every bucket (Work::hist); after ONE scan over the
// concatenated bucket arrays of all indexes this pass builds each row's entry from columns and hashes that already exist and
// drops it straight into its bucket — no temporary entry, no key array.  A bucket's second entry puts the bucket on the
// `multi` list: only those buckets are ordered afterwards (by row id == stable).
template <class RowF>
struct FIdxPlaceDirect {
  RowF rowf;
  u32 *cursor;    // this index's slice of the cursor array (a copy of the scanned bucket array): one atomic yields the position
  IdxEntry *ent;  // shared entry array of the group
  u32 mask;
  GAR_HD void operator()(u32 i) const {
    u64 h = 0;
    IdxEntry e;
    if (!rowf.make(i, &h, &e)) return;
    const u32 k = hash_bucket(h, mask);
#if defined(__CUDA_ARCH__)
    const u32 pos = atomicAdd(&cursor[k], 1u);
#else
    const u32 pos = cursor[k]++;
#endif
    e.tag = hash_tag(h);
    e.row = i;
    ent[pos] = e;
  }
};
// buckets with two or more entries, compacted into a list (one pass over the scanned bucket array; the appends are aggregated
// per warp, so the shared counter sees one atomic per warp, not one per bucket)
struct FIdxMultiList {
  const u32 *begin;
  u32 *multi;  // [0] = count, then bucket ids
  GAR_HD void operator()(u32 b) const {
    const bool m = begin[b + 1] - begin[b] >= 2;
#if defined(__CUDA_ARCH__)
    const unsigned active = __activemask();
    const unsigned votes = __ballot_sync(active, m);
    if (!m) return;
    const unsigned lane = threadIdx.x & 31u;
    const int leader = __ffs(votes) - 1;
    u32 base = 0;
    if ((int)lane == leader) base = atomicAdd(multi, (u32)__popc(votes));
    base = __shfl_sync(votes, base, leader);
    multi[1 + base + __popc(votes & ((1u << lane) - 1u))] = b;
#else
    if (m) multi[1 + multi[0]++] = b;
#endif
  }
};
struct FIdxOrderMulti {
  const u32 *begin;  // the group's whole bucket array (or the owned lists' segment array)
  IdxEntry *ent;
  const u32 *multi;
  u32 *overflow;
  CanonHook canon;
  GAR_HD void operator()(u32 t) const {
    const u32 b = multi[1 + t];
    const u32 lo = begin[b], m = begin[b + 1] - lo;
    if (m > IDX_SMALL_BUCKET) {
      GAR_ATOMIC_ADD(overflow, 1u);
      return;
    }
    for (u32 k = 1; k < m; k++) {  // insertion sort of 32-byte entries by row id, in place
      IdxEntry x = ent[lo + k];
      u32 j = k;
      while (j > 0 && ent[lo + j - 1].row > x.row) {
        ent[lo + j] = ent[lo + j - 1];
        j--;
      }
      if (j != k) ent[lo + j] = x;
    }
    canon(b, ent, lo, m);
  }
};
// everything the host reads back at the END of a diff, gathered into one small block (no read-back in the middle)
enum FlagWord { FW_BAD_KEYS = 0, FW_IDX_OVERFLOW = 1, FW_NDPORTS = 2, FW_NPAIRS = 3, FW_SEC0 = 4 /* 5 section words */, FW_WORDS = 16 };
struct FGatherFinal {
  const u32 *src;
  u32 idx[5];
  const u32 *npairs;  // nullable
  u32 *flags;
  GAR_HD void operator()(u32 k) const {
    if (k < 5) flags[FW_SEC0 + k] = src[idx[k]];
    else if (npairs) flags[FW_NPAIRS] = *npairs;
  }
};
struct FGather5 {
  const u32 *src;
  u32 idx[5];
  const u32 *extra;
  u32 *dst;
  GAR_HD void operator()(u32 k) const { dst[k] = k < 5 ? src[idx[k]] : *extra; }
};
#define GAR_RETRY_WITH_RADIX 1000  // Pipeline::run: rebuild with force_radix (not an error)
#define GAR_REFUSE_EMPTY_CACHE 1001  // orphan deletes against an empty object table (garecon.h "Orphan sweep precondition")
struct FGatherHeader {
  const u32 *ndports;
  u32 *flags;
  GAR_HD void operator()(u32) const { flags[FW_NDPORTS] = *ndports; }
};
// the two per-value joins in one pass (their probe chains overlap: value_joins): first alias record under the value's
// (zone, name), and the object the value names (which also says whether it is an orphan)
struct FValueJoins {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 v) const { value_joins(T, W, v); }
};
// the object half of FValueJoins, alone: re-run after an object delta (the alias links read the actual side only)
struct FResolveValue {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 v) const { resolve_value(T, W, v); }
};
struct FResolveAccel {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 a) const { resolve_accel(T, W, a); }
};
// the load balancer and target-hostname accelerators of each lbIngress row (lbi_resolve): they read the object side's
// tokens and the AWS side's indexes, so they run in both forms of the owner-keyed joins, which follow every change to either
struct FLbiResolve {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 r) const { lbi_resolve(T, W, r); }
};
// owned-list records (payloads: gar_rows.h "index probes"): x < nacc is accelerator x, else owner value x - nacc
GAR_HD IdxEntry own_entry(const DevTables &T, const Work &W, u32 x) {
  IdxEntry e;
  e.tag = e.a0 = e.a1 = 0;
  e.s0 = e.s1 = 0;
  if (x < T.a.n_accels) {
    e.row = x;
    return e;
  }
  const u32 v = x - T.a.n_accels, rec = W.val_rec[v];
  const ValLink l = W.val_link[v];
  e.tag = l.alias_row;
  e.row = v;
  e.a0 = rec;
  e.a1 = W.rec_zone[rec] | ((W.rec_flags[rec] & 1) ? VALNAME_HAS_BACKSLASH : 0u);
  e.s0 = l.alias_dns;
  e.s1 = T.a.rec_name[rec];
  return e;
}
// segment of row x (accelerators first, then values) in the owned lists; 2n: not on any list
GAR_HD u32 own_segment(const DevTables &T, const Work &W, u32 x) {
  const u32 nacc = T.a.n_accels;
  const u32 o = x < nacc ? W.acc_obj[x] : W.val_obj[x - nacc];
  return o == GAR_NONE ? 2 * T.o.n_objects : 2 * o + (x < nacc ? 0u : 1u);
}
// placement into the scanned segments through per-segment cursors (one atomic), rows of a segment in any order: FIdxOrderMulti
// orders the segments with two or more rows afterwards
struct FOwnPlace {
  DevTables T;
  Work W;
  u32 *cursor;
  IdxEntry *ent;
  u32 x0;  // 0: accelerators, n_accels: values
  GAR_HD void operator()(u32 i) const {
    const u32 x = x0 + i, k = own_segment(T, W, x);
    if (k == 2 * T.o.n_objects) return;
#if defined(__CUDA_ARCH__)
    const u32 pos = atomicAdd(&cursor[k], 1u);
#else
    const u32 pos = cursor[k]++;
#endif
    ent[pos] = own_entry(T, W, x);
  }
};
// radix fallback (some list is longer than IDX_SMALL_BUCKET): (segment, x) pairs, stably sorted, then gathered
struct FOwnKeys {
  DevTables T;
  Work W;
  u32 *keys, *vals;
  GAR_HD void operator()(u32 x) const {
    keys[x] = own_segment(T, W, x);
    vals[x] = x;
  }
};
struct FOwnGather {
  DevTables T;
  Work W;
  const u32 *vals;
  const u32 *total;
  IdxEntry *ent;
  GAR_HD void operator()(u32 p) const {
    if (p < *total) ent[p] = own_entry(T, W, vals[p]);
  }
};

// --- count / emit.  counts layout: [GA obj: n][GA orphan: nacc][R53 obj: n][orphan alias: nrec][orphan value: nval][total]
struct CountLayout {
  u32 n, nacc, nrec, nval;
  GAR_HD u32 ga_obj(u32 i) const { return i; }
  GAR_HD u32 ga_orph(u32 a) const { return n + a; }
  GAR_HD u32 r53_obj(u32 i) const { return n + nacc + i; }
  GAR_HD u32 base0() const { return 2 * n + nacc; }
  GAR_HD u32 base1() const { return 2 * n + nacc + nrec; }
  GAR_HD u32 total() const { return 2 * n + nacc + nrec + nval; }
};
// Object sections: every object is evaluated ONCE.  The evaluation writes the status word, the op count and
// up to OPS_STAGE_CAP ops into the object's staging slot; after the scan FCompactOps moves staged ops to their
// final position (objects with more ops than the slot holds are re-evaluated straight into the output).
constexpr u32 OPS_STAGE_CAP = 4;
// `rows` (nullable) selects a subset of object rows (incremental mode): slot t evaluates object rows[t]; status, counts
// and staging are indexed by the slot, everything about the object by its row.
struct FGaObj {
  DevTables T;
  Work W;
  u32 *counts;    // [slots] this section's counts
  gar_op *stage;  // [slots * OPS_STAGE_CAP]
  u32 *status;
  const u32 *rows;
  GAR_HD void operator()(u32 t, bool valid) const {
    u32 i = (rows && valid) ? rows[t] : t;
    OpSink s{stage + (size_t)t * OPS_STAGE_CAP, 0, OPS_STAGE_CAP};
    u32 st = ga_reconcile(T, W, i, valid, s);
    if (valid) {
      status[t] = st;
      counts[t] = s.n;
    }
  }
};
struct FR53Obj {
  DevTables T;
  Work W;
  u32 *counts;
  gar_op *stage;
  u32 *status;
  const u32 *rows;
  GAR_HD void operator()(u32 t, bool valid) const {
    u32 i = (rows && valid) ? rows[t] : t;
    OpSink s{stage + (size_t)t * OPS_STAGE_CAP, 0, OPS_STAGE_CAP};
    // objects finished by r53_prepare keep the status it wrote; every other status is produced here
    u32 prev = (valid && W.r53_mode[i] == R53_MODE_DONE) ? status[t] : 0;
    u32 st = r53_combine(T, W, i, t, valid, prev, s);
    if (valid) {
      status[t] = st;
      counts[t] = s.n;
    }
  }
};
struct FR53Prepare {
  DevTables T;
  Work W;
  u32 *status;
  const u32 *rows;
  GAR_HD void operator()(u32 t, bool valid) const { r53_prepare(T, W, (rows && valid) ? rows[t] : t, t, valid, status); }
};
struct FR53FillPairs {
  DevTables T;
  Work W;
  const u32 *rows;
  GAR_HD void operator()(u32 t) const { r53_fill_pairs(T, W, rows ? rows[t] : t, t); }
};
struct FR53Pair {
  DevTables T;
  Work W;
  GAR_HD void operator()(u32 p, bool valid) const { r53_pair(T, W, p, valid); }
};
// incremental mode: processDelete of one work-queue key that left the cache (globalaccelerator/service.go:28-52,
// route53/service.go:29-46): cleanup of everything the key owns, in the reference's order
struct DelKeys {
  const u8 *kind;
  const gar_str *key;  // refs into `slab`
  const u8 *slab;
};
struct FDelKeyGa {
  DevTables T;
  Work W;
  DelKeys D;
  u32 *counts;   // count pass: written; emit pass: scanned
  gar_op *ops;   // nullptr in the count pass
  u32 cap;
  GAR_HD void operator()(u32 k) const {
    u32 kind = D.kind[k];
    Str key = mkstr(D.slab, D.key[k]);
    if (ops && counts[k + 1] > cap) return;  // beyond the buffer: dropped, the diff is re-run
    OpSink s{ops ? ops + counts[k] : nullptr, 0, 0xFFFFFFFFu};
    OwnerIter it = owner_open(W, key_hash_kinded(kind, key), key);
    for (u32 acc; (acc = owner_next(T, W, kind, it)) != GAR_NONE;) put_delete_chain(T, s, GAR_NONE, 0, acc);
    if (!ops) counts[k] = s.n;
  }
};
struct FDelKeyR53 {
  DevTables T;
  Work W;
  DelKeys D;
  u32 *counts;
  gar_op *ops;
  u32 cap;
  GAR_HD void operator()(u32 k) const {
    u32 kind = D.kind[k];
    Str key = mkstr(D.slab, D.key[k]);
    if (ops && counts[k + 1] > cap) return;
    OpSink s{ops ? ops + counts[k] : nullptr, 0, 0xFFFFFFFFu};
    Owned ow;
    owned_collect(T, W, key_hash_kinded(kind, key), kind, key, ow);
    r53_cleanup(T, W, GAR_NONE, 0, ow, s);
    if (!ops) counts[k] = s.n;
  }
};
struct FRowKnownEg {
  gar_bindings b;
  GAR_HD bool make(u32 i, u64 *h, IdxEntry *e) const {
    *h = gar_hash(mkstr(b.slab, b.known_eg_arn[i]));
    e->a0 = e->a1 = 0;
    e->s0 = b.known_eg_arn[i];
    e->s1 = 0;
    return true;
  }
};
struct FEgb {
  DevTables T;
  Work W;
  DevBindings B;
  u32 *counts;   // count pass: written; emit pass: scanned
  gar_op *ops;
  u32 *status;
  u32 cap;
  GAR_HD void operator()(u32 k) const {
    if (ops && counts[k + 1] > cap) return;
    OpSink s{ops ? ops + counts[k] : nullptr, 0, 0xFFFFFFFFu};
    u32 st = egb_reconcile(T, W, B, k, s);
    if (ops) status[k] = st;
    else counts[k] = s.n;
  }
};
struct FGatherDerived {
  const u32 *derived, *rows;
  u32 *out;
  GAR_HD void operator()(u32 t) const { out[t] = derived[rows[t]] & 0xFFu; }
};
struct FCompactOps {
  DevTables T;
  Work W;
  const u32 *scanned;  // exclusive-scanned counts of this section (entry t+1 exists: the layout is contiguous)
  const gar_op *stage;
  gar_op *ops;
  u32 ctrl;
  const u32 *rows;
  u32 cap;  // capacity of `ops`: nothing is written at or beyond it
  GAR_HD void operator()(u32 t, bool valid) const {
    u32 i = (rows && valid) ? rows[t] : t;
    u32 off = 0, c = 0;
    if (valid) {
      off = scanned[t];
      c = scanned[t + 1] - off;
      if (off > cap || c > cap - off) c = 0;  // does not fit: dropped (the total in the flag block tells the host)
      if (c <= OPS_STAGE_CAP)
        for (u32 k = 0; k < c; k++) ops[off + k] = stage[(size_t)t * OPS_STAGE_CAP + k];
    }
    // objects with more ops than a staging slot holds are re-evaluated straight into the output (warp-uniform:
    // the decide functions vote, so the whole warp enters when any lane needs it)
    bool redo = valid && c > OPS_STAGE_CAP;
    if (GAR_ANY(redo)) {
      OpSink s{ops + off, 0, redo ? c : 0u};
      if (ctrl == GAR_CTRL_GA) ga_reconcile(T, W, i, redo, s);
      else r53_reconcile(T, W, i, redo, s);  // the per-object routine: same decisions as prepare/pairs/combine
    }
  }
};
struct FGaOrphan {
  DevTables T;
  Work W;
  CountLayout L;
  u32 *counts;
  gar_op *ops;
  u32 cap;
  GAR_HD void operator()(u32 a) const {
    if (ops && counts[L.ga_orph(a) + 1] == counts[L.ga_orph(a)]) return;  // emit pass: nothing to write
    if (ops && counts[L.ga_orph(a) + 1] > cap) return;                    // beyond the buffer: dropped, the diff is re-run
    OpSink s{ops ? ops + counts[L.ga_orph(a)] : nullptr, 0, 0xFFFFFFFFu};
    ga_orphan(T, W, a, s);
    if (!ops) counts[L.ga_orph(a)] = s.n;
  }
};
// orphan section order: per zone, alias phase (by record row) then metadata phase (by value row)
struct FR53OrphanAlias {
  DevTables T;
  Work W;
  CountLayout L;
  u32 *counts;
  gar_op *ops;
  u32 cap;
  GAR_HD void operator()(u32 r) const {
    if (!ops) {
      OpSink s{nullptr, 0, 0};
      r53_orphan_alias(T, W, r, s);
      counts[L.base0() + r] = s.n;
      return;
    }
    if (counts[L.base0() + r + 1] == counts[L.base0() + r]) return;
    if (counts[L.total()] > cap) return;  // the R53 orphan section interleaves two count ranges: all or nothing
    u32 z = W.rec_zone[r];
    u32 zv = T.a.rec_val_begin[T.a.zone_rec_begin[z]];  // first value row of the zone
    u32 off = counts[L.base0()] + (counts[L.base1() + zv] - counts[L.base1()]) + (counts[L.base0() + r] - counts[L.base0()]);
    OpSink s{ops + off, 0, 0xFFFFFFFFu};
    r53_orphan_alias(T, W, r, s);
  }
};
struct FR53OrphanValue {
  DevTables T;
  Work W;
  CountLayout L;
  u32 *counts;
  gar_op *ops;
  u32 cap;
  GAR_HD void operator()(u32 v) const {
    if (!ops) {
      counts[L.base1() + v] = W.val_orphan[v];
      return;
    }
    if (!W.val_orphan[v] || counts[L.total()] > cap) return;
    u32 r = W.val_rec[v];
    u32 z = W.rec_zone[r];
    u32 rend = T.a.zone_rec_begin[z + 1];  // alias-phase ops of zones 0..z precede
    u32 off = counts[L.base0()] + (counts[L.base0() + rend] - counts[L.base0()]) + (counts[L.base1() + v] - counts[L.base1()]);
    gar_op o;
    o.head = GAR_OP_HEAD(GAR_OP_R53_DELETE_RECORD, GAR_CTRL_R53, 0);
    o.obj = GAR_NONE;
    o.sub = 1;
    o.a0 = z;
    o.a1 = r;
    o.a2 = v;
    ops[off] = o;
  }
};

// ------------------------------------------------------------------ the pipeline

struct DiffCounts {
  u64 n_ops;
  u64 section_begin[GAR_N_SECTIONS + 1];
  u64 n_dports;
  u32 bad_keys;
};

GAR_HD u32 next_pow2(u32 x) {
  u32 p = 1;
  while (p < x) p <<= 1;
  return p;
}
inline int ilog2(u32 p) {
  int b = 0;
  while ((1u << b) < p) b++;
  return b;
}

template <class B>
struct Pipeline {
  B &be;
  DevTables T;
  Work W{};
  bool force_radix = false;  // set when a bucket exceeded IDX_SMALL_BUCKET in the previous attempt
  explicit Pipeline(B &b, const DevTables &t) : be(b), T(t) {}

  // nb: buckets (power of two).  load: target rows per bucket used to size nb from the row count.
  template <class RowF>
  HashIdx build_index(int slot, u32 nrows, u32 load, RowF rowf, u32 *overflow, bool force_radix, CanonHook canon = {}) {
    u32 nb = next_pow2(nrows / load < 16 ? 16 : nrows / load);
    u32 *keys = (u32 *)be.ensure(S_SORT_KEYS, sizeof(u32) * (size_t)(nrows + 1));
    u32 *vals = (u32 *)be.ensure(S_SORT_VALS, sizeof(u32) * (size_t)(nrows + 1));
    IdxEntry *tmp = (IdxEntry *)be.ensure(S_SORT_TAGS, sizeof(IdxEntry) * (size_t)(nrows + 1));
    u32 *begin = (u32 *)be.ensure(slot + 0, sizeof(u32) * (size_t)(nb + 2));
    IdxEntry *ent = (IdxEntry *)be.ensure(slot + 1, sizeof(IdxEntry) * (size_t)(nrows + 1));
    be.fill32(begin, 0, nb + 2);
    if (nrows) be.for_each("idx_rows", nrows, FIdxRows<RowF>{rowf, keys, force_radix ? vals : nullptr, tmp, begin, nb - 1, nb});
    be.exclusive_scan(begin, nb + 2);  // begin[b] = #rows with key < b; begin[nb] = #indexed rows
    if (nrows && !force_radix) {
      u32 *cursor = (u32 *)be.ensure(S_SORT_KEYS_ALT, sizeof(u32) * (size_t)(nb + 1));
      be.copy32(cursor, begin, nb);
      be.for_each("idx_place", nrows, FIdxPlace{keys, cursor, tmp, ent, nb});
      be.for_each("idx_order", nb, FIdxOrder{begin, ent, overflow, canon});
    } else if (nrows) {
      u32 *keys2 = (u32 *)be.ensure(S_SORT_KEYS_ALT, sizeof(u32) * (size_t)(nrows + 1));
      u32 *vals2 = (u32 *)be.ensure(S_SORT_VALS_ALT, sizeof(u32) * (size_t)(nrows + 1));
      be.sort_pairs(keys, vals, keys2, vals2, nrows, ilog2(nb) + 1);
      be.for_each("idx_gather", nrows, FIdxGather{vals, begin + nb, tmp, ent});
      if (canon.canon) be.for_each("idx_order", nb, FIdxCanon{begin, ent, canon});
    }
    return HashIdx{begin, ent, nb - 1};
  }

  // ---- prepare: everything that depends on the snapshot only (stages 1-3).  Runs once per loaded snapshot; the
  // digests and indexes stay resident for every later diff (full or incremental).
  bool prepared = false;
  u64 n_dports = 0;  // from the final read-back of the last diff
  u32 *errflag = nullptr;

  u32 acc_guest_from = 0xFFFFFFFFu;  // sharded mode: set before prepare()
  u32 sharded = 0;
  bool orphan_sweep = true;        // GAR_FLAG_NO_ORPHANS clears it
  bool allow_empty_cache = false;  // GAR_FLAG_ALLOW_EMPTY_CACHE

  // per-object work arrays (the object side: sized by the object table, rebuilt after an object delta)
  void alloc_obj_work() {
    const u32 n = T.o.n_objects, nlbi = T.o.n_lbi;
    W.derived = (u32 *)be.ensure(S_DERIVED, 4 * (size_t)(n + 1));
    W.okey_hash = (u64 *)be.ensure(S_OKEY_HASH, 8 * (size_t)(n + 1));
    W.ann_r53 = (gar_str *)be.ensure(S_ANN_R53, 8 * (size_t)(n + 1));
    W.ann_name = (gar_str *)be.ensure(S_ANN_NAME, 8 * (size_t)(n + 1));
    W.ann_tags = (gar_str *)be.ensure(S_ANN_TAGS, 8 * (size_t)(n + 1));
    W.ann_listen = (gar_str *)be.ensure(S_ANN_LISTEN, 8 * (size_t)(n + 1));
    W.dport_begin = (u32 *)be.out_dport_begin(n);
    W.tok_code = (u8 *)be.out_tok_code(nlbi);
    W.tok_name = (gar_str *)be.out_tok_name(nlbi);
    W.tok_region = (gar_str *)be.out_tok_region(nlbi);
    W.lbi_res = (LbiRes *)be.ensure(S_LBI_RES, sizeof(LbiRes) * (size_t)(nlbi + 1));
    W.r53_mode = (u8 *)be.ensure(S_R53_MODE, (size_t)n + 1);
    W.r53_acc = (u32 *)be.ensure(S_R53_ACC, 4 * (size_t)(n + 1));
    W.r53_acc_dns = (gar_str *)be.ensure(S_R53_ACC_DNS, 8 * (size_t)(n + 1));
    W.obj_canon = (u32 *)be.ensure(S_OBJ_CANON, 4 * (size_t)(n + 1));
  }
  CanonHook canon_hook(u32 b0, u32 b1) const { return CanonHook{W.obj_canon, T.o.slab, b0, b1}; }
  void alloc_work() {
    const u32 nacc = T.a.n_accels, nrec = T.a.n_records, nval = T.a.n_values;
    alloc_obj_work();
    W.acc_flags = (u32 *)be.ensure(S_ACC_FLAGS, 4 * (size_t)(nacc + 1));
    W.acc_owner_key = (gar_str *)be.ensure(S_ACC_OWNER_KEY, 8 * (size_t)(nacc + 1));
    W.acc_owner = (gar_str *)be.ensure(S_ACC_OWNER, 8 * (size_t)(nacc + 1));
    W.acc_thost = (gar_str *)be.ensure(S_ACC_THOST, 8 * (size_t)(nacc + 1));
    W.acc_managed = (gar_str *)be.ensure(S_ACC_MANAGED, 8 * (size_t)(nacc + 1));
    W.acc_owner_hash = (u64 *)be.ensure(S_ACC_OWNER_HASH, 8 * (size_t)(nacc + 1));
    W.acc_thost_hash = (u64 *)be.ensure(S_ACC_THOST_HASH, 8 * (size_t)(nacc + 1));
    W.rec_name_hash = (u64 *)be.ensure(S_REC_NAME_HASH, 8 * (size_t)(nrec + 1));
    W.val_key_hash = (u64 *)be.ensure(S_VAL_KEY_HASH, 8 * (size_t)(nval + 1));
    W.rec_zone = (u32 *)be.ensure(S_REC_ZONE, 4 * (size_t)(nrec + 1));
    W.val_rec = (u32 *)be.ensure(S_VAL_REC, 4 * (size_t)(nval + 1));
    W.val_cls = (u8 *)be.ensure(S_VAL_CLS, nval + 1);
    W.val_key = (gar_str *)be.ensure(S_VAL_KEY, 8 * (size_t)(nval + 1));
    W.val_orphan = (u8 *)be.ensure(S_VAL_ORPHAN, nval + 1);
    W.val_obj = (u32 *)be.ensure(S_VAL_OBJ, 4 * (size_t)(nval + 1));
    W.acc_obj = (u32 *)be.ensure(S_ACC_OBJ, 4 * (size_t)(nacc + 1));
    W.val_link = (ValLink *)be.ensure(S_VAL_LINK, sizeof(ValLink) * (size_t)(nval + 1));
    W.acc_digest = (AccDigest *)be.ensure(S_ACC_DIGEST, sizeof(AccDigest) * (size_t)(nacc + 1));
    W.lb_hash = (u64 *)be.ensure(S_LB_HASH, 8 * (size_t)(T.a.n_lbs + 1));
    W.rec_flags = (u8 *)be.ensure(S_REC_FLAGS, (size_t)nrec + 1);
    for (int k = 0; k < IX_N; k++) W.hist[k] = IxHist{nullptr, 0};
    W.pair_cap = 0;
    W.dport_cap = 0;
    errflag = (u32 *)be.ensure(S_ERRFLAG, 256);
    be.fill32(errflag, 0, FW_WORDS);
    W.acc_guest_from = acc_guest_from;
    W.sharded = sharded;
  }
  void stage1() {
    const u32 n = T.o.n_objects, nlbi = T.o.n_lbi, nacc = T.a.n_accels, nrec = T.a.n_records, nval = T.a.n_values;
    u32 *derived_public = (u32 *)be.out_derived(n);
    // stage 1: row-local preprocessing
    if (n) be.for_each("classify_objects", n, FClassify{T, W, derived_public, nullptr, errflag});
    if (nlbi) be.for_each_staged("tokenise_hostnames", nlbi, FTokenise{T, W});
    if (nacc) be.for_each("digest_accelerators", nacc, FDigestAccel{T, W});
    if (T.a.n_lbs) be.for_each("hash_load_balancers", T.a.n_lbs, FLbHash{T, W});
    {
      unsigned long long *zm = (unsigned long long *)(errflag + 16 + 8);  // 32 bytes inside the 256-byte flag block, 8-byte aligned
      be.fill32((u32 *)zm, 0, 8);
      if (T.a.n_zones) be.for_each("zone_len_mask", T.a.n_zones, FZoneLenMask{T, W, zm});
      W.zone_len_mask = (const u64 *)zm;
    }
    if (nrec) {  // includes the records' values
      u32 *big = (u32 *)be.ensure(S_SORT_KEYS, 4 * (size_t)(nval / REC_INLINE_VALUES + 2));
      u32 *huge = (u32 *)be.ensure(S_SORT_VALS, 4 * (size_t)(nval / REC_HUGE_VALUES + 2));
      be.fill32(big, 0, 1);
      be.fill32(huge, 0, 1);
      be.for_each_staged("prepare_records", nrec, FPrepareRecord{T, W, big, huge});
      if (nval > REC_INLINE_VALUES) be.for_each("prepare_records", BIG_BLOCKS * 256, FClassifyBigRecords{T, W, big, huge});
    }
  }
  // ---- one-pass index build (the default).  plan: which indexes, their bucket counts and where each one's slice of the
  // shared bucket / entry arrays starts.  The histogram hooks (Work::hist) must be armed BEFORE the row-local passes run.
  struct IxPlan {
    u32 off[IX_N] = {}, nb[IX_N] = {}, rows[IX_N] = {};
    bool want[IX_N] = {};
    u32 total_nb = 0;
    u64 total_rows = 0;
  };
  IxPlan planA;
  u32 *ixa_begin = nullptr, *ixa_fill = nullptr, *ixa_multi = nullptr;
  IdxEntry *ixa_ent = nullptr;
  u32 ovn_nb = 0;
  void arm_group_a(u32 want_mask) {
    const u32 rows[IX_N] = {T.a.n_lbs, T.a.n_accels, T.a.n_accels, T.a.n_zones, T.a.n_values, T.a.n_records, T.o.n_objects, 0};
    const u32 load[IX_N] = {1, 1, 1, 1, 1, 2, 1, 8};
    planA = IxPlan{};
    for (int k = 0; k < IX_OVN; k++) {
      planA.want[k] = (want_mask >> k) & 1u;
      if (!planA.want[k]) continue;
      planA.rows[k] = rows[k];
      planA.nb[k] = next_pow2(rows[k] / load[k] < 16 ? 16 : rows[k] / load[k]);
      planA.off[k] = planA.total_nb;
      planA.total_nb += planA.nb[k];
      planA.total_rows += rows[k];
    }
    ixa_begin = (u32 *)be.ensure(S_IXA_BEGIN, 4 * (size_t)(planA.total_nb + 2));
    be.fill32(ixa_begin, 0, (size_t)planA.total_nb + 2);
    for (int k = 0; k < IX_OVN; k++)
      if (planA.want[k]) W.hist[k] = IxHist{ixa_begin + planA.off[k], planA.nb[k] - 1};
  }
  HashIdx group_a_index(int k) const { return HashIdx{ixa_begin + planA.off[k], ixa_ent, planA.nb[k] - 1}; }
  template <class RowF>
  FIdxPlaceDirect<RowF> placer(int k, RowF rowf) const {
    return FIdxPlaceDirect<RowF>{rowf, ixa_fill + planA.off[k], ixa_ent, planA.nb[k] - 1};
  }
  // scan + place + order of group A (after every armed row pass has run)
  void finish_group_a() {
    u32 *overflow = errflag + FW_IDX_OVERFLOW;
    be.exclusive_scan(ixa_begin, planA.total_nb + 1);  // positions in the shared entry array; [total_nb] = number of entries
    ixa_fill = (u32 *)be.ensure(S_IXA_FILL, 4 * (size_t)(planA.total_nb + 1));  // the placement cursors
    ixa_ent = (IdxEntry *)be.ensure(S_IXA_ENT, sizeof(IdxEntry) * (size_t)(planA.total_rows + 1));
    const u32 multi_cap = (u32)(planA.total_rows / 2 + 1);
    ixa_multi = (u32 *)be.ensure(S_IXA_MULTI, 4 * (size_t)(multi_cap + 2));
    be.copy32(ixa_fill, ixa_begin, (size_t)planA.total_nb + 1);
    be.fill32(ixa_multi, 0, 1);
    const IxPlan &P = planA;
    auto n = [&](int k) { return P.want[k] ? P.rows[k] : 0u; };
    be.for_each_multi("idx_place", {n(IX_LB), n(IX_THOST), n(IX_ZONE), n(IX_ALIAS), n(IX_OBJ), P.total_nb},
                      placer(IX_LB, FRowLb{T, W}), placer(IX_THOST, FRowThost{T, W}), placer(IX_ZONE, FRowZone{T}),
                      placer(IX_ALIAS, FRowAlias{T, W}), placer(IX_OBJ, FRowObj{T, W}), FIdxMultiList{ixa_begin, ixa_multi});
    const CanonHook canon = P.want[IX_OBJ] ? canon_hook(P.off[IX_OBJ], P.off[IX_OBJ] + P.nb[IX_OBJ]) : CanonHook{};
    be.for_each_dyn("idx_order", ixa_multi, multi_cap, FIdxOrderMulti{ixa_begin, ixa_ent, ixa_multi, overflow, canon});
    if (P.want[IX_LB]) W.ix_lb = group_a_index(IX_LB);
    if (P.want[IX_THOST]) W.ix_thost = group_a_index(IX_THOST);
    if (P.want[IX_ZONE]) W.ix_zone = group_a_index(IX_ZONE);
    if (P.want[IX_ALIAS]) W.ix_alias = group_a_index(IX_ALIAS);
    if (P.want[IX_OBJ]) W.ix_obj = group_a_index(IX_OBJ);
  }
  // ---- the owner-keyed joins, resolved from the AWS side (after ix_obj and its obj_canon exist): one fused pass over values
  // (alias links when `link_aliases`, object row, orphan mark) and owner-keyed accelerators (object row) counts the owned-list
  // segments and the buckets of the orphan-value index, whose keys exist only now; then both are built the way group A is:
  // one scan each, one fused placement through cursors, ordering of the segments / buckets with two or more rows.
  // The same launch resolves every lbIngress row's load balancer and target-hostname accelerators (lbi_res): like the owner
  // joins they read both sides of the snapshot, and this is the one step that follows every change to either side.
  void resolve_owners(bool link_aliases) {
    const u32 n = T.o.n_objects, nacc = T.a.n_accels, nval = T.a.n_values, nseg = 2 * n;
    u32 *overflow = errflag + FW_IDX_OVERFLOW;
    W.own_begin = (u32 *)be.ensure(S_OWN_BEGIN, 4 * (size_t)(nseg + 2));
    be.fill32(W.own_begin, 0, (size_t)nseg + 1);
    u32 *ovn = nullptr;
    if (!force_radix) {
      ovn_nb = next_pow2(nval / 8 < 16 ? 16 : nval / 8);
      ovn = (u32 *)be.ensure(S_IX_OVN + 0, 4 * (size_t)(ovn_nb + 2));
      be.fill32(ovn, 0, (size_t)ovn_nb + 2);
      W.hist[IX_OVN] = IxHist{ovn, ovn_nb - 1};
    } else {
      W.hist[IX_OVN] = IxHist{nullptr, 0};
    }
    const u32 nlbi = T.o.n_lbi;
    if (link_aliases) be.for_each_multi("value_joins", {nval, nacc, nlbi}, FValueJoins{T, W}, FResolveAccel{T, W}, FLbiResolve{T, W});
    else be.for_each_multi("resolve_owners", {nval, nacc, nlbi}, FResolveValue{T, W}, FResolveAccel{T, W}, FLbiResolve{T, W});
    be.exclusive_scan(W.own_begin, nseg + 1);  // [nseg] = number of records
    IdxEntry *own = (IdxEntry *)be.ensure(S_OWN_ENT, sizeof(IdxEntry) * ((size_t)nacc + nval + 1));
    if (!force_radix) {
      be.exclusive_scan(ovn, ovn_nb + 1);
      u32 *ovn_cursor = (u32 *)be.ensure(S_OVN_FILL, 4 * (size_t)(ovn_nb + 1));
      IdxEntry *ovn_ent = (IdxEntry *)be.ensure(S_IX_OVN + 1, sizeof(IdxEntry) * (size_t)(nval + 1));
      u32 *ovn_multi = (u32 *)be.ensure(S_OVN_MULTI, 4 * (size_t)(nval / 2 + 3));
      u32 *own_cursor = (u32 *)be.ensure(S_OWN_FILL, 4 * (size_t)(nseg + 1));
      const u32 own_multi_cap = (u32)(((u64)nacc + nval) / 2 + 1);
      u32 *own_multi = (u32 *)be.ensure(S_OWN_MULTI, 4 * (size_t)(own_multi_cap + 2));
      be.copy32(ovn_cursor, ovn, (size_t)ovn_nb + 1);
      be.copy32(own_cursor, W.own_begin, (size_t)nseg + 1);
      be.fill32(ovn_multi, 0, 1);
      be.fill32(own_multi, 0, 1);
      be.for_each_multi("idx_place", {nval, ovn_nb, nacc, nval, nseg}, FIdxPlaceDirect<FRowOvn>{FRowOvn{T, W}, ovn_cursor, ovn_ent, ovn_nb - 1},
                        FIdxMultiList{ovn, ovn_multi}, FOwnPlace{T, W, own_cursor, own, 0}, FOwnPlace{T, W, own_cursor, own, nacc},
                        FIdxMultiList{W.own_begin, own_multi});
      be.for_each_dyn("idx_order", ovn_multi, nval / 2 + 1, FIdxOrderMulti{ovn, ovn_ent, ovn_multi, overflow});
      be.for_each_dyn("idx_order", own_multi, own_multi_cap, FIdxOrderMulti{W.own_begin, own, own_multi, overflow});
      W.ix_ovn = HashIdx{ovn, ovn_ent, ovn_nb - 1};
    } else {  // a list longer than IDX_SMALL_BUCKET: (segment, row) pairs through the stable radix sort
      const u32 nx = nacc + nval;
      u32 *keys = (u32 *)be.ensure(S_SORT_KEYS, 4 * (size_t)(nx + 1));
      u32 *vals = (u32 *)be.ensure(S_SORT_VALS, 4 * (size_t)(nx + 1));
      u32 *keys2 = (u32 *)be.ensure(S_SORT_KEYS_ALT, 4 * (size_t)(nx + 1));
      u32 *vals2 = (u32 *)be.ensure(S_SORT_VALS_ALT, 4 * (size_t)(nx + 1));
      if (nx) {
        be.for_each("own_keys", nx, FOwnKeys{T, W, keys, vals});
        be.sort_pairs(keys, vals, keys2, vals2, nx, ilog2(nseg + 1) + 1);
        be.for_each("own_gather", nx, FOwnGather{T, W, vals, W.own_begin + nseg, own});
      }
      W.ix_ovn = build_index(S_IX_OVN, nval, 8, FRowOvn{T, W}, overflow, true);
    }
    W.own = own;
    owners_stale = false;
  }
  // ix_owner / ix_val: what a key that LEFT the cache owns (gar_diff_keys' deleted keys; objects in the cache read their owned
  // lists).  Built the first time a diff carries deleted keys; they read the AWS side only, so they stay until it changes.
  bool owner_indexes = false;
  void build_owner_indexes() {
    if (owner_indexes) return;
    u32 *overflow = errflag + FW_IDX_OVERFLOW;
    W.ix_owner = build_index(S_IX_OWNER, T.a.n_accels, 1, FRowOwner{T, W}, overflow, force_radix);
    W.ix_val = build_index(S_IX_VAL, T.a.n_values, 1, FRowVal{T, W}, overflow, force_radix);
    owner_indexes = true;
  }

  // what the sharded mode's routing needs of a rank's slice: the row-local pass + the (zone, name) -> alias record index
  void prepare_route() {
    alloc_work();
    arm_group_a(1u << IX_ALIAS);
    stage1();
    finish_group_a();
  }
  // a directory shard's tables (gar_shard.h): probes in lbi_*, load balancers, accelerator stubs.  The probes are answered
  // "first row wins", so every bucket must be in row order: a load-balancer key or target hostname with more rows than
  // IDX_SMALL_BUCKET (left unordered by the per-bucket ordering) rebuilds both indexes through the stable radix sort, as
  // prepare() does after a retry.
  void prepare_directory() {
    alloc_work();
    be.fill32(errflag, 0, FW_WORDS);
    arm_group_a((1u << IX_LB) | (1u << IX_THOST));
    if (T.o.n_lbi) be.for_each("tokenise_hostnames", T.o.n_lbi, FTokenise{T, W});
    if (T.a.n_accels) be.for_each("digest_accelerators", T.a.n_accels, FDigestAccel{T, W});
    if (T.a.n_lbs) be.for_each("hash_load_balancers", T.a.n_lbs, FLbHash{T, W});
    finish_group_a();
    u32 fl[FW_WORDS];
    be.download(fl, errflag, sizeof(fl));
    if (fl[FW_IDX_OVERFLOW]) {
      u32 *overflow = errflag + FW_IDX_OVERFLOW;
      W.ix_lb = build_index(S_IX_LB, T.a.n_lbs, 1, FRowLb{T, W}, overflow, true);
      W.ix_thost = build_index(S_IX_THOST, T.a.n_accels, 1, FRowThost{T, W}, overflow, true);
    }
  }

  u32 dport_cap = 0, pair_cap = 0;  // capacities of the two intermediate relations whose size only the device knows
  u64 ops_cap = 0;
  bool tiny_caps = false;  // test hook (environment GAR_TINY_CAPS=1): start every capacity at 1 so that the grow-and-rerun paths run
  int prepare() {
    const u32 n = T.o.n_objects, nacc = T.a.n_accels, nzone = T.a.n_zones, nrec = T.a.n_records;
    if (T.a.n_lbs > LBI_ROW_MASK || nacc > LBI_ROW_MASK) return GAR_E_INVALID;  // LbiRes keeps these rows in 30 bits
    alloc_work();
    if (!force_radix) arm_group_a((1u << IX_LB) | (1u << IX_THOST) | (1u << IX_ZONE) | (1u << IX_ALIAS) | (1u << IX_OBJ));
    stage1();
    listen_ports();

    // stage 3: hash indexes, then the owner-keyed joins
    u32 *overflow = errflag + FW_IDX_OVERFLOW;
    if (!force_radix) {
      finish_group_a();
    } else {  // some bucket or owned list was too large for the per-bucket ordering: everything through the stable radix sort
      W.ix_lb = build_index(S_IX_LB, T.a.n_lbs, 1, FRowLb{T, W}, overflow, true);
      W.ix_thost = build_index(S_IX_THOST, nacc, 1, FRowThost{T, W}, overflow, true);
      W.ix_zone = build_index(S_IX_ZONE, nzone, 1, FRowZone{T}, overflow, true);
      W.ix_alias = build_index(S_IX_ALIAS, nrec, 2, FRowAlias{T, W}, overflow, true);
      W.ix_obj = build_index(S_IX_OBJ, n, 1, FRowObj{T, W}, overflow, true, canon_hook(0, 0xFFFFFFFFu));
    }
    resolve_owners(true);
    obj_stale = false;
    owner_indexes = false;
    return GAR_OK;
  }
  // stage 2: listen-ports annotation -> desired port lists (count, scan, write).  The total stays on the device: the list
  // buffer has a capacity, a diff that needs more is re-run (run_with)
  void listen_ports() {
    const u32 n = T.o.n_objects;
    be.fill32(W.dport_begin, 0, (size_t)n + 1);
    if (n) be.for_each("listen_ports_count", n, FJsonCount{T, W});
    be.exclusive_scan(W.dport_begin, n + 1);
    be.for_each("gather_header", 1, FGatherHeader{W.dport_begin + n, errflag});
    if (dport_cap < n / 2 + 1024 && !(tiny_caps && dport_cap)) dport_cap = tiny_caps ? 1 : n / 2 + 1024;
    W.dport_cap = dport_cap;
    W.dports = (i32 *)be.out_dports(dport_cap);
    if (n) be.for_each("listen_ports_write", n, FJsonWrite{T, W});
  }

  // ---- object deltas (gar_delta.h).  The prepared state splits in two halves:
  //   actual side  digests, LB hashes, zone mask, records / values, the LB / target-hostname / zone / alias indexes, the
  //                value -> alias links and the on-demand ix_owner / ix_val: depend on the AWS tables only and stay resident
  //                across deltas;
  //   object side  classify, tokenise, listen ports, ix_obj + obj_canon, and the owner-keyed joins that point into the object
  //                rows (val_obj / acc_obj, the owned lists, the orphan value marks + ix_ovn) and the lbIngress rows (lbi_res):
  //                rebuilt over the whole resident table after a delta.
  // obj_stale: the object table changed since the object side was built.  owners_stale: the owner-keyed joins lag behind ix_obj.
  bool obj_stale = false, owners_stale = false;
  void prepare_objects() {
    const u32 n = T.o.n_objects, nlbi = T.o.n_lbi;
    alloc_obj_work();
    be.fill32(errflag, 0, FW_WORDS);
    W.hist[IX_OBJ] = IxHist{nullptr, 0};  // ix_obj is built on its own below: its size no longer fits the fused group-A arrays
    u32 *derived_public = (u32 *)be.out_derived(n);
    if (n) be.for_each("classify_objects", n, FClassify{T, W, derived_public, nullptr, errflag});
    if (nlbi) be.for_each_staged("tokenise_hostnames", nlbi, FTokenise{T, W});
    listen_ports();
    W.ix_obj = build_index(S_IX_OBJ, n, 1, FRowObj{T, W}, errflag + FW_IDX_OVERFLOW, force_radix, canon_hook(0, 0xFFFFFFFFu));
    obj_stale = false;
    owners_stale = true;
  }
  // a complete ix_obj of the current object table (key resolution of a delta), with the same index-overflow fallback as run_with
  int index_objects() {
    for (int attempt = 0; attempt < 2; attempt++) {
      if (!prepared) prepare();
      else if (obj_stale) prepare_objects();
      prepared = true;
      u32 fl[FW_WORDS];
      be.download(fl, errflag, sizeof(fl));
      if (fl[FW_BAD_KEYS]) return GAR_E_INVALID;
      if (fl[FW_IDX_OVERFLOW] && !force_radix) {
        force_radix = true;
        prepared = false;
        continue;
      }
      return GAR_OK;
    }
    return GAR_E_STATE;
  }

  // route53 ensure in relational form over `slots` object slots (rows == nullptr: slot = object row).  The number of
  // (object, hostname) pairs stays on the device: the pair arrays have a capacity (re-run with larger ones if exceeded) and the
  // pair kernel reads its extent from pair_begin[slots].
  u64 n_pairs = 0;  // size of the relation in the last decide (filled from the final read-back; gar_last_counters)
  void r53_relational(u32 slots, const u32 *rows, u32 *st_r53) {
    W.pair_begin = (u32 *)be.ensure(S_PAIR_BEGIN, 4 * (size_t)(slots + 2));
    be.fill32(W.pair_begin, 0, (size_t)slots + 1);
    if (slots) be.for_each_warp("r53_prepare", slots, FR53Prepare{T, W, st_r53, rows});
    be.exclusive_scan(W.pair_begin, slots + 1);
    if (pair_cap < slots + slots / 2 + 1024 && !(tiny_caps && pair_cap)) pair_cap = tiny_caps ? 1 : slots + slots / 2 + 1024;
    W.pair_cap = pair_cap;
    W.pair_obj = (u32 *)be.ensure(S_PAIR_OBJ, 4 * (size_t)(pair_cap + 1));
    W.pair_hn = (gar_str *)be.ensure(S_PAIR_HN, 8 * (size_t)(pair_cap + 1));
    W.pair_code = (u8 *)be.ensure(S_PAIR_CODE, (size_t)pair_cap + 1);
    W.pair_zone = (u32 *)be.ensure(S_PAIR_ZONE, 4 * (size_t)(pair_cap + 1));
    W.pair_rec = (u32 *)be.ensure(S_PAIR_REC, 4 * (size_t)(pair_cap + 1));
    if (slots) {
      be.for_each("r53_fill_pairs", slots, FR53FillPairs{T, W, rows});
      be.for_each_warp_dyn("r53_pairs", W.pair_begin + slots, pair_cap, FR53Pair{T, W});
    }
  }

  // ---- full diff: every object + the orphan sections.  No read-back inside: sizes travel in the flag block (run_with).
  template <class OpsAlloc>
  int decide_all(OpsAlloc ops_alloc) {
    const u32 n = T.o.n_objects, nacc = T.a.n_accels, nrec = T.a.n_records, nval = T.a.n_values;
    // stage 4: evaluate every object once (status + count + staged ops); count the orphan sections
    CountLayout L{n, nacc, nrec, nval};
    u32 *counts = (u32 *)be.ensure(S_COUNTS, 4 * (size_t)(L.total() + 2));
    be.fill32(counts, 0, (size_t)L.total() + 1);
    gar_op *stage_ga = (gar_op *)be.ensure(S_STAGE_GA, sizeof(gar_op) * ((size_t)n * OPS_STAGE_CAP + 1));
    gar_op *stage_r53 = (gar_op *)be.ensure(S_STAGE_R53, sizeof(gar_op) * ((size_t)n * OPS_STAGE_CAP + 1));
    u32 *st_ga = (u32 *)be.out_status_ga(n);
    u32 *st_r53 = (u32 *)be.out_status_r53(n);
    if (n) be.for_each_warp("ga_objects", n, FGaObj{T, W, counts + L.ga_obj(0), stage_ga, st_ga, nullptr});
    r53_relational(n, nullptr, st_r53);
    if (n) be.for_each_warp("r53_objects", n, FR53Obj{T, W, counts + L.r53_obj(0), stage_r53, st_r53, nullptr});
    if (orphan_sweep)
      be.for_each_multi("orphans_count", {nacc, nrec, nval}, FGaOrphan{T, W, L, counts, nullptr, 0}, FR53OrphanAlias{T, W, L, counts, nullptr, 0},
                        FR53OrphanValue{T, W, L, counts, nullptr, 0});
    be.exclusive_scan(counts, L.total() + 1);
    be.for_each("gather_section_begins", 6, FGatherFinal{counts, {0, L.ga_orph(0), L.r53_obj(0), L.base0(), L.total()}, W.pair_begin + n, errflag});

    // stage 5: move ops to their final, canonical positions (writes beyond the buffer's capacity are dropped: the diff is
    // re-run with a larger buffer)
    const u64 est = tiny_caps ? 1 : (u64)n + nacc / 8 + 1024;
    if (ops_cap < est) ops_cap = est;
    gar_op *ops = (gar_op *)ops_alloc(ops_cap);
    const u32 cap = ops_cap > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (u32)ops_cap;
    if (n) be.for_each_warp("ga_objects_compact", n, FCompactOps{T, W, counts + L.ga_obj(0), stage_ga, ops, GAR_CTRL_GA, nullptr, cap});
    if (n) be.for_each_warp("r53_objects_compact", n, FCompactOps{T, W, counts + L.r53_obj(0), stage_r53, ops, GAR_CTRL_R53, nullptr, cap});
    if (orphan_sweep)
      be.for_each_multi("orphans_emit", {nacc, nrec, nval}, FGaOrphan{T, W, L, counts, ops, cap}, FR53OrphanAlias{T, W, L, counts, ops, cap},
                        FR53OrphanValue{T, W, L, counts, ops, cap});
    return GAR_OK;
  }

  // ---- incremental diff: `m` object rows + `nd` deleted keys (device arrays).  counts layout:
  // [GA rows: m][GA deleted keys: nd][R53 rows: m][R53 deleted keys: nd][total]
  template <class OpsAlloc>
  int decide_keys(const u32 *rows, u32 m, DelKeys D, u32 nd, OpsAlloc ops_alloc) {
    const u32 total = 2 * m + 2 * nd;
    u32 *counts = (u32 *)be.ensure(S_COUNTS, 4 * (size_t)(total + 2));
    be.fill32(counts, 0, (size_t)total + 1);
    u32 *c_ga = counts, *c_gad = counts + m, *c_r53 = counts + m + nd, *c_r53d = counts + 2 * m + nd;
    gar_op *stage_ga = (gar_op *)be.ensure(S_STAGE_GA, sizeof(gar_op) * ((size_t)m * OPS_STAGE_CAP + 1));
    gar_op *stage_r53 = (gar_op *)be.ensure(S_STAGE_R53, sizeof(gar_op) * ((size_t)m * OPS_STAGE_CAP + 1));
    u32 *st_ga = (u32 *)be.out_status_ga(m);
    u32 *st_r53 = (u32 *)be.out_status_r53(m);
    u32 *derived_out = (u32 *)be.out_derived_keys(m);
    if (nd) build_owner_indexes();
    if (m) {
      be.for_each("gather_derived", m, FGatherDerived{W.derived, rows, derived_out});
      be.for_each_warp("ga_objects", m, FGaObj{T, W, c_ga, stage_ga, st_ga, rows});
    }
    if (nd) be.for_each("ga_deleted_keys_count", nd, FDelKeyGa{T, W, D, c_gad, nullptr, 0});
    r53_relational(m, rows, st_r53);
    if (m) be.for_each_warp("r53_objects", m, FR53Obj{T, W, c_r53, stage_r53, st_r53, rows});
    if (nd) be.for_each("r53_deleted_keys_count", nd, FDelKeyR53{T, W, D, c_r53d, nullptr, 0});
    be.exclusive_scan(counts, total + 1);
    be.for_each("gather_section_begins", 6, FGatherFinal{counts, {0, m, m + nd, 2 * m + nd, total}, W.pair_begin + m, errflag});
    const u64 est = tiny_caps ? 1 : 2 * (u64)m + 4 * (u64)nd + 256;
    if (ops_cap < est) ops_cap = est;
    gar_op *ops = (gar_op *)ops_alloc(ops_cap);
    const u32 cap = ops_cap > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (u32)ops_cap;
    if (m) be.for_each_warp("ga_objects_compact", m, FCompactOps{T, W, c_ga, stage_ga, ops, GAR_CTRL_GA, rows, cap});
    if (nd) be.for_each("ga_deleted_keys_emit", nd, FDelKeyGa{T, W, D, c_gad, ops, cap});
    if (m) be.for_each_warp("r53_objects_compact", m, FCompactOps{T, W, c_r53, stage_r53, ops, GAR_CTRL_R53, rows, cap});
    if (nd) be.for_each("r53_deleted_keys_emit", nd, FDelKeyR53{T, W, D, c_r53d, ops, cap});
    return GAR_OK;
  }

  // ---- EndpointGroupBinding set-diff over `nb` bindings (device pointers in `b`)
  template <class OpsAlloc>
  int decide_bindings(const gar_bindings &b, OpsAlloc ops_alloc) {
    u32 *overflow = errflag + FW_IDX_OVERFLOW;
    const u32 nb = b.n_bindings;
    DevBindings DB{b, build_index(S_IX_EG, b.n_known_egs, 1, FRowKnownEg{b}, overflow, force_radix)};
    u32 *counts = (u32 *)be.ensure(S_COUNTS, 4 * (size_t)(nb + 2));
    be.fill32(counts, 0, (size_t)nb + 1);
    u32 *st = (u32 *)be.out_status_ga(nb);
    if (nb) be.for_each("egb_count", nb, FEgb{T, W, DB, counts, nullptr, nullptr, 0});
    be.exclusive_scan(counts, nb + 1);
    be.for_each("gather_section_begins", 6, FGatherFinal{counts, {0, nb, nb, nb, nb}, nullptr, errflag});
    const u64 est = tiny_caps ? 1 : 4 * (u64)nb + 256;
    if (ops_cap < est) ops_cap = est;
    gar_op *ops = (gar_op *)ops_alloc(ops_cap);
    const u32 cap = ops_cap > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (u32)ops_cap;
    if (nb) be.for_each("egb_emit", nb, FEgb{T, W, DB, counts, ops, st, cap});
    return GAR_OK;
  }

  // prepare (once per snapshot) + one of the decide flavours, then the ONE read-back of the diff: the flag block with the
  // section sizes and everything that may force another attempt — a hash bucket too large for the per-bucket ordering
  // (-> stable radix build), or an intermediate relation larger than its buffer (-> larger buffer).  Retries are rare:
  // capacities only grow, so a snapshot shape settles after its first diff.
  // `replayable`: the launch sequence of this flavour depends only on the snapshot and the capacities, so the backend may record
  // it once and replay it (a CUDA graph): the full diff.  Incremental / binding diffs take new host inputs every time.
  int last_launch_mode = 0;  // graph_begin's answer for the last attempt of the last diff (0 for partial diffs; gar_last_counters)
  template <class DecideF>
  int run_with(DiffCounts *dc, bool full, DecideF decide) {
    last_launch_mode = 0;
    for (int attempt = 0; attempt < 8; attempt++) {
      u64 sig = 0;
      if (full) {
        sig = hmix(hmix(prepared ? (obj_stale || owners_stale ? 9 : 1) : 2, force_radix ? 3 : 4), hmix(hmix(dport_cap, pair_cap), ops_cap));
        sig = hmix(sig, hmix(orphan_sweep ? 5 : 6, tiny_caps ? 7 : 8)) | 1;
      }
      const int g = full ? be.graph_begin(sig) : 0;
      last_launch_mode = g;
      int rc = GAR_OK;
      if (g != 2) {
        if (!prepared) rc = prepare();
        else if (obj_stale) prepare_objects();
        if (rc == GAR_OK && owners_stale) resolve_owners(false);  // the decide functions of every flavour read the owned lists
        if (rc == GAR_OK) rc = decide();
      }
      prepared = true;
      if (full) be.graph_end();
      if (rc != GAR_OK) return rc;
      u32 fl[FW_WORDS];
      be.download(fl, errflag, sizeof(fl));
      if (fl[FW_BAD_KEYS]) return GAR_E_INVALID;
      if (fl[FW_IDX_OVERFLOW] && !force_radix) {
        force_radix = true;
        prepared = false;
        continue;
      }
      if (fl[FW_NDPORTS] > dport_cap) {
        dport_cap = fl[FW_NDPORTS] + fl[FW_NDPORTS] / 8 + 16;
        prepared = false;
        continue;
      }
      if (fl[FW_NPAIRS] > pair_cap) {
        pair_cap = fl[FW_NPAIRS] + fl[FW_NPAIRS] / 8 + 16;
        continue;
      }
      const u64 nops = fl[FW_SEC0 + 4];
      if (nops > ops_cap) {
        ops_cap = nops + nops / 8 + 16;
        continue;
      }
      n_dports = fl[FW_NDPORTS];
      n_pairs = fl[FW_NPAIRS];
      for (int k = 0; k < 5; k++) dc->section_begin[k] = fl[FW_SEC0 + k];
      dc->n_ops = nops;
      dc->n_dports = full ? n_dports : 0;
      // an EMPTY object table with owned resources left: an unsynced informer looks exactly like this, and the orphan sections
      // would delete everything the cluster owns.  (A shard that happens to home no object is fine: the cluster is not empty.)
      if (full && T.o.n_objects == 0 && !sharded && !allow_empty_cache && nops != 0) return GAR_REFUSE_EMPTY_CACHE;
      return GAR_OK;
    }
    return GAR_E_STATE;
  }
  template <class OpsAlloc>
  int run(DiffCounts *dc, OpsAlloc ops_alloc) {
    return run_with(dc, true, [&] { return decide_all(ops_alloc); });
  }
  template <class OpsAlloc>
  int run_keys(const u32 *rows, u32 m, DelKeys D, u32 nd, DiffCounts *dc, OpsAlloc ops_alloc) {
    return run_with(dc, false, [&] { return decide_keys(rows, m, D, nd, ops_alloc); });
  }
  template <class OpsAlloc>
  int run_bindings(const gar_bindings &b, DiffCounts *dc, OpsAlloc ops_alloc) {
    return run_with(dc, false, [&] { return decide_bindings(b, ops_alloc); });
  }
};

// ------------------------------------------------------------------ read set (gar_read_set, include/garecon.h)
//
// Backend: for_each, fill32, exclusive_scan(u64 *), download, and read_set_buf(k, bytes) — scratch that no recorded launch
// sequence holds, so the call grows it without dropping the full diff's graph (the 64-bit scan keeps its own tile states too).
// The record read set (gar_read_records) is the same run with `records` set: other items, one bitmap over record rows.
// Steps: prepare as gar_diff_keys does (Pipeline::run_with) -> items per key, scan -> mark (one thread per item) -> popcount
// per bitmap word, scan -> emit rows ascending, zeroing every word read: the bitmaps are all zero between calls, so a call
// costs O(keys + items + table rows / 32).  After a failed call they are cleared again before they are trusted.
GAR_HD u32 popc32(u32 v) {
#if defined(__CUDA_ARCH__)
  return (u32)__popc(v);
#else
  return (u32)__builtin_popcount(v);
#endif
}
struct FReadSetCount {
  DevTables T;
  Work W;
  const u32 *rows;
  u32 m;
  DelKeys D;
  Cursor *cur;  // [2 nd]
  u64 *items;   // [m + nd + 1]
  bool recs;    // the record read set (gar_read_records)
  GAR_HD void operator()(u32 t) const {
    if (t < m) items[t] = recs ? read_records_row_items(W, rows[t]) : read_set_row_items(T, W, rows[t]);
    else if (recs) items[t] = read_records_deleted_items(W, D.kind[t - m], mkstr(D.slab, D.key[t - m]), cur + 2 * (t - m));
    else items[t] = read_set_deleted_items(W, D.kind[t - m], mkstr(D.slab, D.key[t - m]), cur + 2 * (t - m));
  }
};
struct FReadSetMark {
  DevTables T;
  Work W;
  const u32 *rows;
  u32 m, nkeys;
  DelKeys D;
  const Cursor *cur;
  const u64 *items;  // exclusive-scanned
  u64 base;
  ReadSetBits B;
  bool recs;
  GAR_HD void operator()(u32 x) const {
    const u64 q = base + x;
    u32 lo = 0, hi = nkeys;  // the last key whose first item is <= q (a key with no items shares its offset with the next)
    while (hi - lo > 1) {
      const u32 mid = (lo + hi) >> 1;
      if (items[mid] <= q) lo = mid;
      else hi = mid;
    }
    const u32 r = (u32)(q - items[lo]);
    if (lo < m) {
      if (recs) read_records_row_item(T, W, B, rows[lo], r);
      else read_set_row_item(T, W, B, rows[lo], r);
    } else if (recs) {
      read_records_deleted_item(T, W, B, D.kind[lo - m], mkstr(D.slab, D.key[lo - m]), cur + 2 * (lo - m), r);
    } else {
      read_set_deleted_item(T, W, B, D.kind[lo - m], mkstr(D.slab, D.key[lo - m]), cur + 2 * (lo - m), r);
    }
  }
};
struct FReadSetPopc {
  const u32 *bits;
  u64 *cnt;
  GAR_HD void operator()(u32 w) const { cnt[w] = popc32(bits[w]); }
};
struct FReadSetSizes {
  const u64 *cnt;
  ReadSetBits B;
  u64 *sizes;  // [RS_N + 1]: the scanned count at the first word of each bitmap, and the total
  GAR_HD void operator()(u32 s) const { sizes[s] = cnt[B.wb[s]]; }
};
struct ReadSetOut {
  u32 *rows[RS_N];  // ascending rows per bitmap (RS_MISS: lbIngress rows, before the expansion below)
  u32 *miss_obj, *miss_j;
  gar_str *miss_name, *miss_region;
};
struct FReadSetEmit {
  DevTables T;
  Work W;
  const u64 *cnt;
  ReadSetBits B;
  ReadSetOut O;
  GAR_HD void operator()(u32 w) const {
    u32 v = B.bits[w];
    if (!v) return;
    B.bits[w] = 0;
    u32 s = 0;
    while (w >= B.wb[s + 1]) s++;
    u64 pos = cnt[w] - cnt[B.wb[s]];
    for (; v; v &= v - 1, pos++) {
      const u32 r = (w - B.wb[s]) * 32 + ctz64(v);
      if (s != RS_MISS) {
        O.rows[s][pos] = r;
        continue;
      }
      u32 lo = 0, hi = T.o.n_objects;  // the object row whose lbIngress range holds r
      while (hi - lo > 1) {
        const u32 mid = (lo + hi) >> 1;
        if (T.o.obj_lbi_begin[mid] <= r) lo = mid;
        else hi = mid;
      }
      O.miss_obj[pos] = lo;
      O.miss_j[pos] = r - T.o.obj_lbi_begin[lo];
      O.miss_name[pos] = W.tok_name[r];
      O.miss_region[pos] = W.tok_region[r];
    }
  }
};

// the bitmap buffer last cleared and how many of its words are known to be zero; kept by the engine between calls
struct ReadSetClean {
  u32 *bits = nullptr;
  u32 words = 0;
};
template <class Be, class Pipe>
struct ReadSetter {
  Be &be;
  Pipe &P;
  ReadSetClean &clean;
  bool records = false;  // gar_read_records: only the record bitmap (RS_REC) is sized and filled
  enum { RB_ITEMS, RB_CUR, RB_BITS, RB_CNT, RB_SIZES, RB_OUT32, RB_OUT64, RB_N };
  // rows of each bitmap (RS_N) and the size of each, device pointers valid until the next call
  ReadSetOut out;
  u32 n[RS_N];
  int run(const u32 *rows, u32 m, DelKeys D, u32 nd) {
    DiffCounts dc{};
    int rc = P.run_with(&dc, false, [&] {
      if (nd) P.build_owner_indexes();
      return GAR_OK;
    });
    if (rc != GAR_OK) return rc;
    const DevTables &T = P.T;
    const Work &W = P.W;
    const u32 nk = m + nd;
    u64 *items = (u64 *)be.read_set_buf(RB_ITEMS, 8 * ((size_t)nk + 2));
    Cursor *cur = (Cursor *)be.read_set_buf(RB_CUR, sizeof(Cursor) * (2 * (size_t)nd + 1));
    const u32 size[RS_N] = {records ? 0 : T.a.n_lbs, records ? 0 : T.a.n_accels, records ? 0 : T.a.n_zones, records ? 0 : T.o.n_lbi,
                            records ? T.a.n_records : 0};
    ReadSetBits B;
    B.wb[0] = 0;
    for (int s = 0; s < RS_N; s++) B.wb[s + 1] = B.wb[s] + (size[s] + 31) / 32;
    const u32 nw = B.wb[RS_N];
    B.bits = (u32 *)be.read_set_buf(RB_BITS, 4 * ((size_t)nw + 1));
    if (B.bits != clean.bits || nw > clean.words) be.fill32(B.bits, 0, nw);  // a new buffer, or the last call did not finish
    clean.bits = B.bits;
    clean.words = 0;

    if (nk) be.for_each("read_set_count", nk, FReadSetCount{T, W, rows, m, D, cur, items, records});
    be.fill32((u32 *)(items + nk), 0, 2);
    be.exclusive_scan(items, nk + 1);
    u64 total = 0;
    be.download(&total, items + nk, 8);
    constexpr u64 CHUNK = 1ull << 30;
    for (u64 b = 0; b < total; b += CHUNK)
      be.for_each("read_set_mark", (u32)(total - b < CHUNK ? total - b : CHUNK), FReadSetMark{T, W, rows, m, nk, D, cur, items, b, B, records});

    u64 *cnt = (u64 *)be.read_set_buf(RB_CNT, 8 * ((size_t)nw + 2));
    u64 *sizes = (u64 *)be.read_set_buf(RB_SIZES, 8 * (RS_N + 1));
    if (nw) be.for_each("read_set_popcount", nw, FReadSetPopc{B.bits, cnt});
    be.fill32((u32 *)(cnt + nw), 0, 2);
    be.exclusive_scan(cnt, nw + 1);
    be.for_each("read_set_sizes", RS_N + 1, FReadSetSizes{cnt, B, sizes});
    u32 *o32 = (u32 *)be.read_set_buf(RB_OUT32, 4 * ((size_t)size[0] + size[1] + size[2] + 2 * (size_t)size[3] + size[4] + 1));
    gar_str *o64 = (gar_str *)be.read_set_buf(RB_OUT64, 8 * (2 * (size_t)size[3] + 1));
    out.rows[RS_LB] = o32;
    out.rows[RS_ACC] = o32 + size[0];
    out.rows[RS_ZONE] = out.rows[RS_ACC] + size[1];
    out.rows[RS_MISS] = nullptr;
    out.miss_obj = out.rows[RS_ZONE] + size[2];
    out.miss_j = out.miss_obj + size[3];
    out.rows[RS_REC] = out.miss_j + size[3];
    out.miss_name = o64;
    out.miss_region = o64 + size[3];
    if (nw) be.for_each("read_set_emit", nw, FReadSetEmit{T, W, cnt, B, out});
    u64 sz[RS_N + 1];
    be.download(sz, sizes, sizeof(sz));
    for (int s = 0; s < RS_N; s++) n[s] = (u32)(sz[s + 1] - sz[s]);
    clean.words = nw;
    return GAR_OK;
  }
};
