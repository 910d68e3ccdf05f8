// gar_delta.h — object deltas (gar_snapshot_apply_objects): informer events applied to the resident object table.
//
// Shared by the CUDA backend (gar_engine.cu) and the host simulation (tests/hostsim), like gar_shard.h: functors for the
// data-parallel steps plus a driver template, Splicer<B>, that runs them over a Backend.  Data movement of one delta:
//   1. the keys of the delta (deletes, then upserts) are resolved against the resident ix_obj index on the device, one
//      thread per key with a full key compare after the tag (as find_object does);
//   2. the host turns the resolved rows into the delete / swap-move / replace / append sequence of include/garecon.h:
//      O(batch) work that yields a short list of (new row <- source) overrides on top of the identity map;
//   3. the upsert table is copied to the device; its slab is appended to the resident object slab (16-byte aligned);
//   4. the object table is re-laid out dense into the standby column set: source map, per-row child counts + one scan per
//      CSR, then a gather of the fixed-width columns and a warp-cooperative copy of the child rows (string references of
//      rows that come from the upsert batch are rebased by the slab offset).  The standby set then becomes the resident one.
// Re-laying instead of keeping (begin, end) pairs per row means every decision kernel keeps reading x_begin[i + 1] and
// gar_rows.h does not change.  The pipeline's object side is marked stale and rebuilt by the next diff (gar_pipeline.h).
//
// Backend interface, on top of gar_pipeline.h's:
//   void upload(void *dev_dst, const void *host_src, size_t bytes);
//   void *delta_scratch(int k, size_t bytes);          // staging buffer k (DS_*)
//   void *delta_col(int c, size_t bytes);              // column c (DC_*) of the STANDBY object column set
//   void delta_swap();                                 // the standby set becomes the resident one
//   u8 *delta_slab(u64 keep, u64 need);                // resident object slab with >= need bytes, the first `keep` preserved
//   void *delta_actual_col(int c, size_t bytes);       // the standby buffer of AWS column c (AC_*): not the resident one
//   void delta_actual_swap(int c);                     // column c's standby buffer becomes the resident one
//   u8 *delta_actual_slab(u64 keep, u64 need);         // the same as delta_slab, for the resident AWS slab
//
// AWS deltas (gar_snapshot_apply_actual, ActualSplicer below) re-lay only the AWS families a delta touches — load balancers;
// accelerator -> tag / listener -> port range / listener -> endpoint group -> endpoint; zone -> record -> value — with one
// generic step per parent -> child link, order preserving.  They drop the whole prepared state (the caller does).  Zone
// deltas (gar_snapshot_apply_zones) run on the same splicer: a source map of the zone table with deletes and positioned
// inserts (FDeltaZoneMap), then the same re-layout of zone -> record -> value, zone names included.
#pragma once

#include <stddef.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "gar_pipeline.h"

// object table columns, in gar_objects order (also the order in which gar_snapshot_load uploads them)
enum DeltaCol {
  DC_KIND, DC_SPEC, DC_FLAGS, DC_NS, DC_NAME, DC_ICLS, DC_ANN_B, DC_LBI_B, DC_PORT_B, DC_ANN_KEY, DC_ANN_VAL, DC_LBI_HOST, DC_PORT_NUM,
  DC_PORT_PROTO, DC_N
};
// AWS table columns, in gar_actual order (also the order in which gar_snapshot_load uploads them)
enum ActualCol {
  AC_LB_REGION, AC_LB_NAME, AC_LB_DNS, AC_LB_ARN, AC_LB_STATE, AC_ACC_NAME, AC_ACC_DNS, AC_ACC_ENABLED, AC_ACC_TAG_B, AC_ACC_LIS_B, AC_TAG_KEY,
  AC_TAG_VAL, AC_LIS_PROTO, AC_LIS_PR_B, AC_LIS_EG_B, AC_PR_FROM, AC_EG_EP_B, AC_EP_ID, AC_ZONE_NAME, AC_ZONE_REC_B, AC_REC_NAME, AC_REC_TYPE,
  AC_REC_ALIAS, AC_REC_ALIAS_DNS, AC_REC_VAL_B, AC_VAL_VALUE, AC_N
};
// AWS tables
enum ActualTable { AT_LB, AT_ACC, AT_TAG, AT_LIS, AT_PR, AT_EG, AT_EP, AT_ZONE, AT_REC, AT_VAL, AT_N };
// staging buffers: the upsert columns (DS_UP + DC_*), keys, source map; for AWS deltas the delta rows (DS_A_UP + AC_*), a
// source map per table (DS_A_SRC + AT_*), the deleted / (new row, source) lists of the root tables and the zone-name check.
// DS_A_COL + 2 * c (+ 1): the two buffers AWS column c alternates between, for a backend that keeps them with its staging
// buffers (the host simulation; the CUDA engine has column sets of its own)
enum DeltaScratch {
  DS_UP = 0, DS_KEY_KIND = DC_N, DS_KEY_REF, DS_KEY_SLAB, DS_COUNTS, DS_OFFS, DS_ROWS, DS_PAIRS, DS_SRC, DS_TOTALS,
  DS_A_UP, DS_A_SRC = DS_A_UP + AC_N, DS_A_DEL = DS_A_SRC + AT_N, DS_A_PAIRS = DS_A_DEL + AT_N, DS_A_ZTARGET = DS_A_PAIRS + AT_N, DS_A_ZREF,
  DS_A_ZSLAB, DS_A_FLAG, DS_A_COL, DS_N = DS_A_COL + 2 * AC_N
};

constexpr u32 SRC_UPSERT = 0x80000000u;  // source map: row of the upsert batch (else a row of the resident table)

// all rows of the resident table that carry key k (kind + "ns/name"); count pass (rows == nullptr), then write pass.
// Entries of an ix_obj bucket are ordered by row, so the rows come out ascending.
struct FDeltaResolve {
  DevTables T;
  HashIdx ix;
  const u8 *kind;
  const gar_str *key;
  const u8 *slab;
  u32 *counts;
  const u32 *offs;
  u32 *rows;
  GAR_HD void operator()(u32 k) const {
    const u32 kd = kind[k];
    const Str ks = mkstr(slab, key[k]);
    Cursor c = idx_open(ix, key_hash_kinded(kd, ks));
    IdxEntry e;
    u32 m = 0;
    while (idx_next(ix, c, &e))
      if (e.a0 == kd && streq(mkstr(T.o.slab, e.s0), ks)) {
        if (rows) rows[offs[k] + m] = e.row;
        m++;
      }
    if (!rows) counts[k] = m;
  }
};
struct FDeltaIdentity {
  u32 *src;
  GAR_HD void operator()(u32 i) const { src[i] = i; }
};
struct FDeltaScatter {
  const u32 *pairs;  // (new row, source) pairs
  u32 *src;
  GAR_HD void operator()(u32 k) const { src[pairs[2 * k]] = pairs[2 * k + 1]; }
};
// the output side of a splice: the standby columns
struct DeltaOut {
  u8 *kind, *spec, *flags;
  gar_str *ns, *name, *icls;
  u32 *ann_b, *lbi_b, *port_b;
  gar_str *ann_key, *ann_val, *lbi_host, *port_proto;
  i32 *port_num;
};
// new row i: fixed-width columns from its source row, and its child counts (row n: the 0 that becomes the scans' total)
struct FDeltaRows {
  gar_objects R, U;  // resident table, upsert batch (device copies)
  const u32 *src;
  u64 base;          // slab offset of the upsert batch's strings
  u32 n;
  DeltaOut D;
  GAR_HD void operator()(u32 i) const {
    if (i == n) {
      D.ann_b[n] = D.lbi_b[n] = D.port_b[n] = 0;
      return;
    }
    const u32 s = src[i], r = s & ~SRC_UPSERT;
    const bool up = (s & SRC_UPSERT) != 0;
    const gar_objects &S = up ? U : R;
    const u64 rb = up ? base : 0;
    const u8 fl = S.obj_flags[r];
    D.kind[i] = S.obj_kind[r];
    D.spec[i] = S.obj_spec_type[r];
    D.flags[i] = fl;
    D.ns[i] = S.obj_ns[r] + rb;  // the offset lives in the low bits of a gar_str
    D.name[i] = S.obj_name[r] + rb;
    D.icls[i] = (fl & GAR_OBJ_HAS_INGRESS_CLASS) ? S.obj_ingress_class[r] + rb : S.obj_ingress_class[r];
    D.ann_b[i] = S.obj_ann_begin[r + 1] - S.obj_ann_begin[r];
    D.lbi_b[i] = S.obj_lbi_begin[r + 1] - S.obj_lbi_begin[r];
    D.port_b[i] = S.obj_port_begin[r + 1] - S.obj_port_begin[r];
  }
};
struct FDeltaTotals {
  const u32 *ann, *lbi, *port;  // the scanned begins' last entries
  u32 *out;
  GAR_HD void operator()(u32) const {
    out[0] = *ann;
    out[1] = *lbi;
    out[2] = *port;
  }
};
// child rows: 32 consecutive threads (one warp on the GPU) per new row, striding over its children — a row with many
// annotations or hostnames is not walked by one thread (DESIGN.md §4 "Skew")
struct FDeltaChildren {
  gar_objects R, U;
  const u32 *src;
  u64 base;
  DeltaOut D;
  GAR_HD void operator()(u32 t) const {
    const u32 i = t >> 5, lane = t & 31u;
    const u32 s = src[i], r = s & ~SRC_UPSERT;
    const bool up = (s & SRC_UPSERT) != 0;
    const gar_objects &S = up ? U : R;
    const u64 rb = up ? base : 0;
    {
      const u32 d0 = D.ann_b[i], c = D.ann_b[i + 1] - d0, s0 = S.obj_ann_begin[r];
      for (u32 k = lane; k < c; k += 32) {
        D.ann_key[d0 + k] = S.ann_key[s0 + k] + rb;
        D.ann_val[d0 + k] = S.ann_val[s0 + k] + rb;
      }
    }
    {
      const u32 d0 = D.lbi_b[i], c = D.lbi_b[i + 1] - d0, s0 = S.obj_lbi_begin[r];
      for (u32 k = lane; k < c; k += 32) D.lbi_host[d0 + k] = S.lbi_hostname[s0 + k] + rb;
    }
    {
      const u32 d0 = D.port_b[i], c = D.port_b[i + 1] - d0, s0 = S.obj_port_begin[r];
      for (u32 k = lane; k < c; k += 32) {
        D.port_num[d0 + k] = S.port_number[s0 + k];
        D.port_proto[d0 + k] = S.port_proto[s0 + k] + rb;
      }
    }
  }
};

// ------------------------------------------------------------------ AWS deltas: one generic step per parent -> child link
// Every AWS table is re-laid by the same three functors.  A table's new rows come from a source map (resident row, or
// SRC_UPSERT | row of the delta table); per CSR link the new begins are the children counts + one scan, and the children's
// source map is written one warp per parent; then the child table is re-laid from that map, level by level.

// survivors of an order-preserving delete: new row j <- resident row j + #{deleted rows before it}.  key[m] = d_m - m for
// the deleted rows d ascending: the number of survivors ahead of the m-th deleted row, so the shift is #{m : key[m] <= j}
struct FDeltaCompact {
  const u32 *key;
  u32 nd;
  u32 *src;
  GAR_HD void operator()(u32 j) const {
    u32 lo = 0, hi = nd;
    while (lo < hi) {
      const u32 mid = (lo + hi) >> 1;
      if (key[mid] <= j) lo = mid + 1;
      else hi = mid;
    }
    src[j] = j + lo;
  }
};
// new row i of a table: its fixed-width columns from its source row; string references of delta rows rebased by `base`
struct DeltaGatherCol {
  const u8 *r, *u;  // resident column, delta column
  u8 *d;            // standby column
  u32 width, str;
};
struct FDeltaGather {
  const u32 *src;
  u64 base;
  u32 ncols;
  DeltaGatherCol c[5];
  GAR_HD void operator()(u32 i) const {
    const u32 s = src[i], r = s & ~SRC_UPSERT;
    const bool up = (s & SRC_UPSERT) != 0;
    for (u32 k = 0; k < ncols; k++) {
      const DeltaGatherCol &g = c[k];
      const u8 *S = up ? g.u : g.r;
      if (g.width == 1) g.d[i] = S[r];
      else if (g.width == 4) ((u32 *)g.d)[i] = ((const u32 *)S)[r];
      else ((u64 *)g.d)[i] = ((const u64 *)S)[r] + (up && g.str ? base : 0);  // the offset lives in the low bits of a gar_str
    }
  }
};
// child counts of new parent i (row n: the 0 that becomes the scan's total)
struct FDeltaCsrCounts {
  const u32 *src, *rb, *ub;  // parent source map, resident begins, delta begins
  u32 n;
  u32 *db;
  GAR_HD void operator()(u32 i) const {
    if (i == n) {
      db[n] = 0;
      return;
    }
    const u32 s = src[i], r = s & ~SRC_UPSERT;
    const u32 *b = (s & SRC_UPSERT) ? ub : rb;
    db[i] = b[r + 1] - b[r];
  }
};
// the children's source map: 32 consecutive threads (one warp on the GPU) per new parent, striding over its children — a TXT
// set of 10^5 values is not walked by one thread (DESIGN.md §4 "Skew")
struct FDeltaCsrChildren {
  const u32 *src, *rb, *ub, *db;
  u32 *csrc;
  GAR_HD void operator()(u32 t) const {
    const u32 i = t >> 5, lane = t & 31u;
    const u32 s = src[i], r = s & ~SRC_UPSERT, flag = s & SRC_UPSERT;
    const u32 s0 = (flag ? ub : rb)[r], d0 = db[i], c = db[i + 1] - d0;
    for (u32 k = lane; k < c; k += 32) csrc[d0 + k] = flag | (s0 + k);
  }
};
// delta zone k must carry the name of resident zone target[k]
struct FDeltaZoneName {
  const u8 *rslab;
  const gar_str *rname;
  const u32 *target;
  const u8 *dslab;
  const gar_str *dname;
  u32 *bad;
  GAR_HD void operator()(u32 k) const {
    if (!streq(mkstr(rslab, rname[target[k]]), mkstr(dslab, dname[k]))) *bad = 1;
  }
};
// #{m : a[m] < x} for a ascending
GAR_HD u32 delta_rank(const u32 *a, u32 n, u32 x) {
  u32 lo = 0, hi = n;
  while (lo < hi) {
    const u32 mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
// source map of the zone table after a zone delta (include/garecon.h "zone deltas"): thread r < n places resident zone r
// unless it is deleted, thread n + k new zone k, each at the row the header's formula gives.  del: the deleted rows
// ascending; at: added_at (non-decreasing)
struct FDeltaZoneMap {
  const u32 *del, *at;
  u32 nd, na, n;
  u32 *src;
  GAR_HD void operator()(u32 t) const {
    if (t < n) {
      const u32 d = delta_rank(del, nd, t);
      if (d < nd && del[d] == t) return;
      src[t - d + delta_rank(at, na, t + 1)] = t;
    } else {
      const u32 k = t - n, a = at[k];
      src[a - delta_rank(del, nd, a) + k] = SRC_UPSERT | k;
    }
  }
};
// record deltas (include/garecon.h "record deltas") run FDeltaZoneMap over the record table (del: deleted record rows, at: rec_at)
// and re-lay record -> value; the zone table keeps its rows and gets new begins from these counts + one scan.  Zone z's new count:
// its resident records, minus the deleted ones inside its range, plus the records of the delta zone that targets it (target
// strictly ascending, ub: the delta's zone_rec_begin).  Zone row n: the 0 that becomes the scan's total
struct FDeltaRecZoneCounts {
  const u32 *rb, *del, *target, *ub;
  u32 nd, nt, n;
  u32 *db;
  GAR_HD void operator()(u32 z) const {
    if (z == n) {
      db[n] = 0;
      return;
    }
    u32 c = rb[z + 1] - rb[z] - (delta_rank(del, nd, rb[z + 1]) - delta_rank(del, nd, rb[z]));
    const u32 k = delta_rank(target, nt, z);
    if (k < nt && target[k] == z) c += ub[k + 1] - ub[k];
    db[z] = c;
  }
};
// the records of delta zone k must be placed inside its resident zone: rec_at within [rb[z], rb[z + 1]] for z = target[k] (rec_at
// is non-decreasing, checked on the host, so the first and the last record of the zone decide)
struct FDeltaRecAt {
  const u32 *rb, *target, *ub, *at;
  u32 *bad;
  GAR_HD void operator()(u32 k) const {
    const u32 k0 = ub[k], k1 = ub[k + 1], z = target[k];
    if (k0 < k1 && (at[k0] < rb[z] || at[k1 - 1] > rb[z + 1])) *bad = 1;
  }
};

// column layout of gar_actual: table, element width, gar_str or not, and the child table of a begin column (AT_N: none)
struct ActualColInfo {
  u8 table, width, str, child;
  size_t field;
};
#define GAR_AC(t, w, s, ch, f) ActualColInfo{t, w, s, ch, offsetof(gar_actual, f)}
static const ActualColInfo kActualCols[AC_N] = {
    GAR_AC(AT_LB, 8, 1, AT_N, lb_region),          GAR_AC(AT_LB, 8, 1, AT_N, lb_name),          GAR_AC(AT_LB, 8, 1, AT_N, lb_dns),
    GAR_AC(AT_LB, 8, 1, AT_N, lb_arn),             GAR_AC(AT_LB, 1, 0, AT_N, lb_state),         GAR_AC(AT_ACC, 8, 1, AT_N, acc_name),
    GAR_AC(AT_ACC, 8, 1, AT_N, acc_dns),           GAR_AC(AT_ACC, 1, 0, AT_N, acc_enabled),     GAR_AC(AT_ACC, 4, 0, AT_TAG, acc_tag_begin),
    GAR_AC(AT_ACC, 4, 0, AT_LIS, acc_lis_begin),   GAR_AC(AT_TAG, 8, 1, AT_N, tag_key),         GAR_AC(AT_TAG, 8, 1, AT_N, tag_val),
    GAR_AC(AT_LIS, 1, 0, AT_N, lis_proto),         GAR_AC(AT_LIS, 4, 0, AT_PR, lis_pr_begin),   GAR_AC(AT_LIS, 4, 0, AT_EG, lis_eg_begin),
    GAR_AC(AT_PR, 4, 0, AT_N, pr_from),            GAR_AC(AT_EG, 4, 0, AT_EP, eg_ep_begin),     GAR_AC(AT_EP, 8, 1, AT_N, ep_id),
    GAR_AC(AT_ZONE, 8, 1, AT_N, zone_name),        GAR_AC(AT_ZONE, 4, 0, AT_REC, zone_rec_begin), GAR_AC(AT_REC, 8, 1, AT_N, rec_name),
    GAR_AC(AT_REC, 1, 0, AT_N, rec_type),          GAR_AC(AT_REC, 1, 0, AT_N, rec_has_alias),   GAR_AC(AT_REC, 8, 1, AT_N, rec_alias_dns),
    GAR_AC(AT_REC, 4, 0, AT_VAL, rec_val_begin),   GAR_AC(AT_VAL, 8, 1, AT_N, val_value)};
#undef GAR_AC
static const size_t kActualRows[AT_N] = {offsetof(gar_actual, n_lbs),         offsetof(gar_actual, n_accels), offsetof(gar_actual, n_tags),
                                         offsetof(gar_actual, n_listeners),   offsetof(gar_actual, n_port_ranges), offsetof(gar_actual, n_egs),
                                         offsetof(gar_actual, n_endpoints),   offsetof(gar_actual, n_zones),  offsetof(gar_actual, n_records),
                                         offsetof(gar_actual, n_values)};
static const char *const kActualColName[AC_N] = {
    "lb_region", "lb_name", "lb_dns", "lb_arn", "lb_state", "acc_name", "acc_dns", "acc_enabled", "acc_tag_begin", "acc_lis_begin", "tag_key", "tag_val", "lis_proto",
    "lis_pr_begin", "lis_eg_begin", "pr_from", "eg_ep_begin", "ep_id", "zone_name", "zone_rec_begin", "rec_name", "rec_type", "rec_has_alias", "rec_alias_dns",
    "rec_val_begin", "val_value"};
inline const void *&actual_col(gar_actual &a, int c) { return *(const void **)((char *)&a + kActualCols[c].field); }
inline const void *actual_col(const gar_actual &a, int c) { return *(const void *const *)((const char *)&a + kActualCols[c].field); }
inline u32 &actual_rows(gar_actual &a, int t) { return *(u32 *)((char *)&a + kActualRows[t]); }
inline u32 actual_rows(const gar_actual &a, int t) { return *(const u32 *)((const char *)&a + kActualRows[t]); }

// ------------------------------------------------------------------ host-side checks of the (small) upsert batch

// the checks gar_snapshot_load runs on the device, for a table the host holds; "" = valid
inline std::string delta_check_upserts(const gar_objects &o) {
  const u32 n = o.n_objects;
  if (!n) return "";
  if (!o.obj_kind || !o.obj_spec_type || !o.obj_flags || !o.obj_ns || !o.obj_name || !o.obj_ingress_class || !o.obj_ann_begin || !o.obj_lbi_begin ||
      !o.obj_port_begin || (o.n_ann && (!o.ann_key || !o.ann_val)) || (o.n_lbi && !o.lbi_hostname) || (o.n_ports && (!o.port_number || !o.port_proto)) ||
      (o.slab_len && !o.slab))
    return "upserts: NULL column";
  auto str_ok = [&](gar_str r) { return GAR_STR_OFF(r) + GAR_STR_LEN(r) <= o.slab_len; };
  auto csr_ok = [&](const u32 *b, u32 nchildren) {
    if (b[0] != 0 || b[n] != nchildren) return false;
    for (u32 i = 0; i < n; i++)
      if (b[i + 1] < b[i]) return false;
    return true;
  };
  if (!csr_ok(o.obj_ann_begin, o.n_ann)) return "upserts: obj_ann_begin: CSR is not monotone, does not start at 0 or does not end at the child count";
  if (!csr_ok(o.obj_lbi_begin, o.n_lbi)) return "upserts: obj_lbi_begin: CSR is not monotone, does not start at 0 or does not end at the child count";
  if (!csr_ok(o.obj_port_begin, o.n_ports)) return "upserts: obj_port_begin: CSR is not monotone, does not start at 0 or does not end at the child count";
  for (u32 i = 0; i < n; i++) {
    if (o.obj_kind[i] > GAR_KIND_INGRESS || o.obj_spec_type[i] > GAR_SVC_EXTERNALNAME) return "upserts: obj_kind / obj_spec_type out of range";
    if (!str_ok(o.obj_ns[i]) || !str_ok(o.obj_name[i])) return "upserts: obj_ns / obj_name: string reference outside the slab";
    if ((o.obj_flags[i] & GAR_OBJ_HAS_INGRESS_CLASS) && !str_ok(o.obj_ingress_class[i])) return "upserts: obj_ingress_class: string reference outside the slab";
    const u64 sep = GAR_STR_OFF(o.obj_ns[i]) + GAR_STR_LEN(o.obj_ns[i]);
    if (GAR_STR_OFF(o.obj_name[i]) != sep + 1 || sep >= o.slab_len || o.slab[sep] != '/')
      return "upserts: objects layout rule violated: obj_ns and obj_name must be slices of one \"ns/name\" key string";
  }
  for (u32 k = 0; k < o.n_ann; k++)
    if (!str_ok(o.ann_key[k]) || !str_ok(o.ann_val[k])) return "upserts: ann_key / ann_val: string reference outside the slab";
  for (u32 k = 0; k < o.n_lbi; k++)
    if (!str_ok(o.lbi_hostname[k])) return "upserts: lbi_hostname: string reference outside the slab";
  for (u32 k = 0; k < o.n_ports; k++)
    if (!str_ok(o.port_proto[k])) return "upserts: port_proto: string reference outside the slab";
  return "";
}

// the checks gar_snapshot_load runs on an actual table, for the rows of an AWS delta; "" = valid
inline std::string delta_check_actual(const gar_actual &a) {
  if (a.slab_len && !a.slab) return "rows: NULL slab";
  for (int c = 0; c < AC_N; c++) {
    const ActualColInfo &ci = kActualCols[c];
    const u32 n = actual_rows(a, ci.table);
    const void *col = actual_col(a, c);
    const std::string name = std::string("rows: ") + kActualColName[c];
    if (ci.child != AT_N) {
      if (!col) return name + " is NULL";
      const u32 *b = (const u32 *)col;
      bool ok = b[0] == 0 && b[n] == actual_rows(a, ci.child);
      for (u32 i = 0; ok && i < n; i++) ok = b[i + 1] >= b[i];
      if (!ok) return name + ": CSR is not monotone, does not start at 0 or does not end at the child count";
      continue;
    }
    if (!n) continue;
    if (!col) return name + " is NULL";
    if (ci.str) {
      const gar_str *s = (const gar_str *)col;
      for (u32 i = 0; i < n; i++)
        if (GAR_STR_OFF(s[i]) + GAR_STR_LEN(s[i]) > a.slab_len) return name + ": string reference outside the slab";
    }
  }
  auto enum_ok = [](const u8 *col, u32 n, u32 max_value) {
    for (u32 i = 0; i < n; i++)
      if (col[i] > max_value) return false;
    return true;
  };
  if (!enum_ok(a.lb_state, a.n_lbs, GAR_LB_FAILED)) return "rows: lb_state out of range";
  if (!enum_ok(a.lis_proto, a.n_listeners, GAR_PROTO_UDP)) return "rows: lis_proto out of range";
  if (!enum_ok(a.rec_type, a.n_records, GAR_RR_AAAA)) return "rows: rec_type out of range";
  return "";
}

// ------------------------------------------------------------------ the driver

// B: the backend the splice runs on; PB: the backend of the engine's Pipeline (the same one, unless B adds the delta buffers
// to an existing backend, as the host simulation does)
template <class B, class PB = B>
struct Splicer {
  B &be;
  Pipeline<PB> &P;
  DevTables &T;  // the resident tables: T.o is replaced by a splice
  std::string error;

  template <class Tp>
  const Tp *up(int k, const Tp *host, size_t count) {
    const size_t bytes = count * sizeof(Tp);
    void *p = be.delta_scratch(k, bytes + GAR_SLAB_PAD + 16);
    if (bytes) be.upload(p, host, bytes);
    return (const Tp *)p;
  }

  // GAR_OK, GAR_E_INVALID (error says why; nothing changed) or another gar_rc
  int apply(const gar_object_delta &d, gar_delta_result &out) {
    static const gar_objects kNoUpserts{};
    const gar_objects &U = (d.upserts && d.upserts->n_objects) ? *d.upserts : kNoUpserts;
    const u32 nu = U.n_objects, nd = d.n_deleted, nk = nd + nu;
    if ((nu && !out.upsert_row) || (nd && (!out.deleted_row || !out.moved_from))) return invalid("NULL result array");
    if (nd && (!d.deleted_kind || !d.deleted_key)) return invalid("NULL deleted-key arrays");
    error = delta_check_upserts(U);
    if (!error.empty()) return GAR_E_INVALID;
    // the keys, deletes first: kind + "ns/name" in one host slab; every key at most once
    std::vector<u8> kind(nk + 1, 0), kslab;
    std::vector<gar_str> kref(nk + 1, 0);
    std::unordered_set<std::string> seen;
    for (u32 k = 0; k < nk; k++) {
      const char *p;
      size_t len;
      if (k < nd) {
        if (!d.deleted_key[k] || d.deleted_kind[k] > GAR_KIND_INGRESS) return invalid("bad deleted key");
        kind[k] = d.deleted_kind[k];
        p = d.deleted_key[k];
        len = strlen(p);
      } else {
        const u32 u = k - nd;
        kind[k] = U.obj_kind[u];
        p = (const char *)U.slab + GAR_STR_OFF(U.obj_ns[u]);
        len = GAR_STR_LEN(U.obj_ns[u]) + 1 + GAR_STR_LEN(U.obj_name[u]);
      }
      std::string key(1, (char)('0' + kind[k]));
      key.append(p, len);
      if (!seen.insert(key).second) return invalid("a key appears twice in one delta (deletes and upserts together): coalesce the events first");
      kref[k] = GAR_STR(kslab.size(), len);
      kslab.insert(kslab.end(), p, p + len);
    }
    const u64 base = nu ? (T.o.slab_len + 15) & ~(u64)15 : 0;
    if (nu && base + U.slab_len + GAR_SLAB_PAD >= (1ull << GAR_STR_OFF_BITS)) return invalid("the resident object slab would outgrow 2^40 bytes: reload");
    if ((u64)T.o.n_objects + nu >= (1u << 27)) return invalid("too many objects for one snapshot");
    out.n_objects = T.o.n_objects;
    out.slab_base = base;
    out.slab_len = T.o.slab_len;
    if (!nk) return GAR_OK;

    // 1. resolve every key against ix_obj: all rows that carry it, ascending
    int rc = P.index_objects();
    if (rc != GAR_OK) return invalid("the resident object table could not be indexed");
    kslab.resize(kslab.size() + GAR_SLAB_PAD, 0);
    const u8 *dkind = up(DS_KEY_KIND, kind.data(), nk);
    const gar_str *dref = up(DS_KEY_REF, kref.data(), nk);
    const u8 *dkslab = up(DS_KEY_SLAB, kslab.data(), kslab.size());
    u32 *dcounts = (u32 *)be.delta_scratch(DS_COUNTS, 4 * (size_t)(nk + 1));
    be.for_each("delta_resolve", nk, FDeltaResolve{T, P.W.ix_obj, dkind, dref, dkslab, dcounts, nullptr, nullptr});
    std::vector<u32> counts(nk), offs(nk + 1, 0);
    be.download(counts.data(), dcounts, 4 * (size_t)nk);
    for (u32 k = 0; k < nk; k++) offs[k + 1] = offs[k] + counts[k];
    std::vector<u32> match(offs[nk] + 1);
    if (offs[nk]) {
      const u32 *doffs = up(DS_OFFS, offs.data(), nk + 1);
      u32 *drows = (u32 *)be.delta_scratch(DS_ROWS, 4 * (size_t)(offs[nk] + 1));
      be.for_each("delta_resolve", nk, FDeltaResolve{T, P.W.ix_obj, dkind, dref, dkslab, dcounts, doffs, drows});
      be.download(match.data(), drows, 4 * (size_t)offs[nk]);
    }

    // 2. the delete / move / replace / append sequence (include/garecon.h), on rows of the resident table ("orig" rows)
    u32 n = T.o.n_objects;
    std::unordered_map<u32, u32> orig_at, cur_of;  // moved rows only: current row -> orig row, orig row -> current row
    std::unordered_set<u32> gone;                  // orig rows deleted
    auto lowest = [&](u32 k) {
      u32 best = GAR_NONE;
      for (u32 m = offs[k]; m < offs[k + 1]; m++) {
        const u32 o = match[m];
        if (gone.count(o)) continue;
        auto it = cur_of.find(o);
        best = std::min(best, it == cur_of.end() ? o : it->second);
      }
      return best;
    };
    auto orig = [&](u32 row) {
      auto it = orig_at.find(row);
      return it == orig_at.end() ? row : it->second;
    };
    for (u32 k = 0; k < nd; k++) {
      const u32 r = lowest(k);
      out.deleted_row[k] = r;
      out.moved_from[k] = GAR_NONE;
      if (r == GAR_NONE) continue;
      const u32 last = n - 1, o_r = orig(r);
      gone.insert(o_r);
      cur_of.erase(o_r);
      if (r != last) {
        const u32 o_last = orig(last);
        orig_at[r] = o_last;
        cur_of[o_last] = r;
        out.moved_from[k] = last;
      }
      orig_at.erase(last);
      n--;
    }
    std::unordered_map<u32, u32> src_at(orig_at.begin(), orig_at.end());  // new row -> source, where not the identity
    for (u32 u = 0; u < nu; u++) {
      u32 r = lowest(nd + u);
      if (r == GAR_NONE) r = n++;
      src_at[r] = SRC_UPSERT | u;
      out.upsert_row[u] = r;
    }
    out.n_objects = n;
    if (src_at.empty() && n == T.o.n_objects) return GAR_OK;  // only absent keys: nothing moves

    // 3. the upsert batch on the device; its strings behind the resident ones
    gar_objects DU{};
    u8 *slab = (u8 *)T.o.slab;
    u64 slab_len = T.o.slab_len;
    if (nu) {
      DU = U;
      DU.obj_kind = up(DS_UP + DC_KIND, U.obj_kind, nu);
      DU.obj_spec_type = up(DS_UP + DC_SPEC, U.obj_spec_type, nu);
      DU.obj_flags = up(DS_UP + DC_FLAGS, U.obj_flags, nu);
      DU.obj_ns = up(DS_UP + DC_NS, U.obj_ns, nu);
      DU.obj_name = up(DS_UP + DC_NAME, U.obj_name, nu);
      DU.obj_ingress_class = up(DS_UP + DC_ICLS, U.obj_ingress_class, nu);
      DU.obj_ann_begin = up(DS_UP + DC_ANN_B, U.obj_ann_begin, nu + 1);
      DU.obj_lbi_begin = up(DS_UP + DC_LBI_B, U.obj_lbi_begin, nu + 1);
      DU.obj_port_begin = up(DS_UP + DC_PORT_B, U.obj_port_begin, nu + 1);
      DU.ann_key = up(DS_UP + DC_ANN_KEY, U.ann_key, U.n_ann);
      DU.ann_val = up(DS_UP + DC_ANN_VAL, U.ann_val, U.n_ann);
      DU.lbi_hostname = up(DS_UP + DC_LBI_HOST, U.lbi_hostname, U.n_lbi);
      DU.port_number = up(DS_UP + DC_PORT_NUM, U.port_number, U.n_ports);
      DU.port_proto = up(DS_UP + DC_PORT_PROTO, U.port_proto, U.n_ports);
      slab_len = base + U.slab_len;
      slab = be.delta_slab(T.o.slab_len, slab_len + GAR_SLAB_PAD);
      static const u8 kZeros[GAR_SLAB_PAD] = {};
      if (U.slab_len) be.upload(slab + base, U.slab, U.slab_len);
      be.upload(slab + slab_len, kZeros, GAR_SLAB_PAD);
    }
    gar_objects R = T.o;
    R.slab = slab;

    // 4. the dense re-layout into the standby set
    std::vector<u32> pairs;
    pairs.reserve(2 * src_at.size());
    for (auto &kv : src_at) {
      pairs.push_back(kv.first);
      pairs.push_back(kv.second);
    }
    u32 *dsrc = (u32 *)be.delta_scratch(DS_SRC, 4 * (size_t)(n + 1));
    if (n) be.for_each("delta_source_map", n, FDeltaIdentity{dsrc});
    if (!pairs.empty()) be.for_each("delta_source_map", (u32)src_at.size(), FDeltaScatter{up(DS_PAIRS, pairs.data(), pairs.size()), dsrc});
    DeltaOut D{};
    D.kind = (u8 *)be.delta_col(DC_KIND, (size_t)n + 16);
    D.spec = (u8 *)be.delta_col(DC_SPEC, (size_t)n + 16);
    D.flags = (u8 *)be.delta_col(DC_FLAGS, (size_t)n + 16);
    D.ns = (gar_str *)be.delta_col(DC_NS, 8 * (size_t)n + 16);
    D.name = (gar_str *)be.delta_col(DC_NAME, 8 * (size_t)n + 16);
    D.icls = (gar_str *)be.delta_col(DC_ICLS, 8 * (size_t)n + 16);
    D.ann_b = (u32 *)be.delta_col(DC_ANN_B, 4 * (size_t)(n + 1) + 16);
    D.lbi_b = (u32 *)be.delta_col(DC_LBI_B, 4 * (size_t)(n + 1) + 16);
    D.port_b = (u32 *)be.delta_col(DC_PORT_B, 4 * (size_t)(n + 1) + 16);
    be.for_each("delta_rows", n + 1, FDeltaRows{R, DU, dsrc, base, n, D});
    be.exclusive_scan(D.ann_b, n + 1);
    be.exclusive_scan(D.lbi_b, n + 1);
    be.exclusive_scan(D.port_b, n + 1);
    u32 *dtot = (u32 *)be.delta_scratch(DS_TOTALS, 64);
    be.for_each("delta_totals", 1, FDeltaTotals{D.ann_b + n, D.lbi_b + n, D.port_b + n, dtot});
    u32 tot[3];
    be.download(tot, dtot, sizeof(tot));
    D.ann_key = (gar_str *)be.delta_col(DC_ANN_KEY, 8 * (size_t)tot[0] + 16);
    D.ann_val = (gar_str *)be.delta_col(DC_ANN_VAL, 8 * (size_t)tot[0] + 16);
    D.lbi_host = (gar_str *)be.delta_col(DC_LBI_HOST, 8 * (size_t)tot[1] + 16);
    D.port_num = (i32 *)be.delta_col(DC_PORT_NUM, 4 * (size_t)tot[2] + 16);
    D.port_proto = (gar_str *)be.delta_col(DC_PORT_PROTO, 8 * (size_t)tot[2] + 16);
    if (n) be.for_each("delta_children", n * 32, FDeltaChildren{R, DU, dsrc, base, D});
    be.delta_swap();
    gar_objects &O = T.o;
    O.n_objects = n;
    O.obj_kind = D.kind;
    O.obj_spec_type = D.spec;
    O.obj_flags = D.flags;
    O.obj_ns = D.ns;
    O.obj_name = D.name;
    O.obj_ingress_class = D.icls;
    O.obj_ann_begin = D.ann_b;
    O.obj_lbi_begin = D.lbi_b;
    O.obj_port_begin = D.port_b;
    O.n_ann = tot[0];
    O.ann_key = D.ann_key;
    O.ann_val = D.ann_val;
    O.n_lbi = tot[1];
    O.lbi_hostname = D.lbi_host;
    O.n_ports = tot[2];
    O.port_number = D.port_num;
    O.port_proto = D.port_proto;
    O.slab = slab;
    O.slab_len = slab_len;
    P.T = T;
    P.obj_stale = true;
    out.slab_len = slab_len;
    return GAR_OK;
  }

 private:
  int invalid(const char *msg) {
    error = msg;
    return GAR_E_INVALID;
  }
};

// ------------------------------------------------------------------ the AWS-delta driver
// The order-preserving splice of include/garecon.h "AWS deltas".  The host checks the (small) delta and turns the targets
// into a source map of each root table (LBs, accelerators, zones); only the families a delta touches are then re-laid into
// standby columns by relayout(), level by level.  Nothing resident changes before the last level is written: the standby
// columns become the resident ones at the end (delta_actual_swap).  The caller drops the pipeline's prepared state.
template <class B>
struct ActualSplicer {
  B &be;
  DevTables &T;  // the resident tables: T.a is replaced by a splice
  std::string error;
  gar_actual R{}, U{}, N{};  // resident table, delta rows (device copies), the table being built
  u64 base = 0;
  bool written[AC_N] = {};
  bool move_zones = false;  // a zone delta: zone rows move, so zone_name is re-laid with the record lists

  // GAR_OK, GAR_E_INVALID (error says why; nothing changed) or another gar_rc
  int apply(const gar_actual_delta &d, gar_actual_delta_result &out) {
    const gar_actual no_rows = empty_table();
    const gar_actual &H = d.rows ? *d.rows : no_rows;
    R = T.a;
    error = delta_check_actual(H);
    if (!error.empty()) return GAR_E_INVALID;
    if ((H.n_lbs && !d.lb_target) || (H.n_accels && !d.acc_target) || (H.n_zones && !d.zone_target) || (d.n_lb_deleted && !d.lb_deleted) ||
        (d.n_acc_deleted && !d.acc_deleted))
      return invalid("NULL target or deleted-row array");
    std::vector<u32> lb_key, lb_pairs, acc_key, acc_pairs, zone_pairs;
    u32 n_lbs = 0, n_accels = 0;
    if (!plan("load balancer", R.n_lbs, H.n_lbs, d.lb_target, d.n_lb_deleted, d.lb_deleted, lb_key, lb_pairs, n_lbs)) return GAR_E_INVALID;
    if (!plan("accelerator", R.n_accels, H.n_accels, d.acc_target, d.n_acc_deleted, d.acc_deleted, acc_key, acc_pairs, n_accels)) return GAR_E_INVALID;
    if (n_accels >= (1u << 27)) return invalid("too many accelerators for one snapshot");
    {
      std::unordered_set<u32> seen;
      for (u32 k = 0; k < H.n_zones; k++) {
        const u32 z = d.zone_target[k];
        if (z >= R.n_zones) return invalid("zone_target out of range (adding hosted zones is a reload)");
        if (!seen.insert(z).second) return invalid("a zone appears twice in zone_target");
        zone_pairs.push_back(z);
        zone_pairs.push_back(SRC_UPSERT | k);
      }
    }
    const bool has_rows = H.n_lbs || H.n_accels || H.n_zones;  // (a table without them has no children: its CSRs end at 0)
    base = has_rows ? (R.slab_len + 15) & ~(u64)15 : 0;
    if (has_rows && base + H.slab_len + GAR_SLAB_PAD >= (1ull << GAR_STR_OFF_BITS)) return invalid("the resident AWS slab would outgrow 2^40 bytes: reload");
    if (H.n_zones && !zone_names_match(H, d.zone_target)) return invalid("a delta zone's zone_name differs from the name of the resident zone it replaces");
    N = R;
    const bool lbs = H.n_lbs || d.n_lb_deleted, accs = H.n_accels || d.n_acc_deleted;
    if (lbs || accs || H.n_zones) {
      stage(H, has_rows);
      int rc = GAR_OK;
      if (lbs) rc = relayout(AT_LB, root_map(AT_LB, n_lbs, lb_key, lb_pairs), n_lbs);
      if (rc == GAR_OK && accs) rc = relayout(AT_ACC, root_map(AT_ACC, n_accels, acc_key, acc_pairs), n_accels);
      if (rc == GAR_OK && H.n_zones) rc = relayout(AT_ZONE, root_map(AT_ZONE, R.n_zones, {}, zone_pairs), R.n_zones);
      if (rc != GAR_OK) return rc;
      for (int c = 0; c < AC_N; c++)
        if (written[c]) be.delta_actual_swap(c);
      T.a = N;
    }
    out.n_lbs = T.a.n_lbs;
    out.n_accels = T.a.n_accels;
    out.n_tags = T.a.n_tags;
    out.n_listeners = T.a.n_listeners;
    out.n_port_ranges = T.a.n_port_ranges;
    out.n_egs = T.a.n_egs;
    out.n_endpoints = T.a.n_endpoints;
    out.n_records = T.a.n_records;
    out.n_values = T.a.n_values;
    out.slab_base = base;
    out.slab_len = T.a.slab_len;
    return GAR_OK;
  }

  // the zone-set splice of include/garecon.h "zone deltas": the host checks the delta, FDeltaZoneMap writes the zone table's
  // source map, and relayout() re-lays zone -> record -> value.  GAR_OK, GAR_E_INVALID (error says why; nothing changed) or
  // another gar_rc
  int apply(const gar_zone_delta &d, gar_zone_delta_result &out) {
    const gar_actual no_rows = empty_table();
    const gar_actual &H = d.added ? *d.added : no_rows;
    R = T.a;
    if (H.n_lbs || H.n_accels || H.n_tags || H.n_listeners || H.n_port_ranges || H.n_egs || H.n_endpoints)
      return invalid("added: a zone delta carries hosted zones and their records only, no load balancer or accelerator rows");
    error = delta_check_actual(H);
    if (!error.empty()) return GAR_E_INVALID;
    const u32 n = R.n_zones, na = H.n_zones, nd = d.n_deleted;
    if ((na && !d.added_at) || (nd && !d.deleted)) return invalid("NULL added_at or deleted array");
    for (u32 k = 0; k < na; k++) {
      if (d.added_at[k] > n) return invalid("added_at out of range");
      if (k && d.added_at[k] < d.added_at[k - 1]) return invalid("added_at decreases");
    }
    std::vector<u32> del(d.deleted, d.deleted + nd);
    std::sort(del.begin(), del.end());
    for (u32 m = 0; m < nd; m++) {
      if (del[m] >= n) return invalid("deleted zone row out of range");
      if (m && del[m] == del[m - 1]) return invalid("a zone row appears twice in deleted");
    }
    if ((u64)n - nd + na >= (1u << 27)) return invalid("too many zones for one snapshot");
    const u32 n_new = n - nd + na;
    base = na ? (R.slab_len + 15) & ~(u64)15 : 0;
    if (na && base + H.slab_len + GAR_SLAB_PAD >= (1ull << GAR_STR_OFF_BITS)) return invalid("the resident AWS slab would outgrow 2^40 bytes");
    N = R;
    if (na || nd) {
      stage(H, na != 0);
      u32 *src = (u32 *)be.delta_scratch(DS_A_SRC + AT_ZONE, 4 * (size_t)(n_new + 1));
      if (n + na)
        be.for_each("delta_zone_map", n + na,
                    FDeltaZoneMap{(const u32 *)up(DS_A_DEL + AT_ZONE, del.data(), 4 * (size_t)nd), (const u32 *)up(DS_A_PAIRS + AT_ZONE, d.added_at, 4 * (size_t)na), nd, na, n, src});
      move_zones = true;
      const int rc = relayout(AT_ZONE, src, n_new);
      if (rc != GAR_OK) return rc;
      for (int c = 0; c < AC_N; c++)
        if (written[c]) be.delta_actual_swap(c);
      T.a = N;
    }
    out.n_zones = T.a.n_zones;
    out.n_records = T.a.n_records;
    out.n_values = T.a.n_values;
    out.slab_base = base;
    out.slab_len = T.a.slab_len;
    return GAR_OK;
  }

  // the record splice of include/garecon.h "record deltas": the host checks the delta's own order (O(delta)), two small kernels
  // check its zones against the resident ones, FDeltaZoneMap writes the record table's source map, FDeltaRecZoneCounts + a scan
  // give zone_rec_begin, and relayout() re-lays record -> value.  GAR_OK, GAR_E_INVALID (error says why; nothing changed) or
  // another gar_rc
  int apply(const gar_record_delta &d, gar_record_delta_result &out) {
    const gar_actual no_rows = empty_table();
    const gar_actual &H = d.rows ? *d.rows : no_rows;
    R = T.a;
    if (H.n_lbs || H.n_accels || H.n_tags || H.n_listeners || H.n_port_ranges || H.n_egs || H.n_endpoints)
      return invalid("rows: a record delta carries zones with their record sets only, no load balancer or accelerator rows");
    error = delta_check_actual(H);
    if (!error.empty()) return GAR_E_INVALID;
    const u32 n = R.n_records, nz = H.n_zones, ni = H.n_records, nd = d.n_deleted;
    if ((nz && !d.zone_target) || (ni && !d.rec_at) || (nd && !d.deleted)) return invalid("NULL zone_target, rec_at or deleted array");
    for (u32 k = 0; k < nz; k++) {
      if (d.zone_target[k] >= R.n_zones) return invalid("zone_target out of range (adding hosted zones is gar_snapshot_apply_zones)");
      if (k && d.zone_target[k] <= d.zone_target[k - 1]) return invalid("zone_target is not strictly ascending");
    }
    for (u32 k = 0; k < ni; k++) {
      if (d.rec_at[k] > n) return invalid("rec_at out of range");
      if (k && d.rec_at[k] < d.rec_at[k - 1]) return invalid("rec_at decreases");
    }
    std::vector<u32> del(d.deleted, d.deleted + nd);
    std::sort(del.begin(), del.end());
    for (u32 m = 0; m < nd; m++) {
      if (del[m] >= n) return invalid("deleted record row out of range");
      if (m && del[m] == del[m - 1]) return invalid("a record row appears twice in deleted");
    }
    if ((u64)n - nd + ni >= (1u << 27)) return invalid("too many records for one snapshot");
    const u32 n_new = n - nd + ni;
    base = ni ? (R.slab_len + 15) & ~(u64)15 : 0;
    if (ni && base + H.slab_len + GAR_SLAB_PAD >= (1ull << GAR_STR_OFF_BITS)) return invalid("the resident AWS slab would outgrow 2^40 bytes");
    const u32 *target = nullptr, *at = nullptr;
    if (nz) {
      const u32 zero[2] = {0, 0};
      u32 *bad = (u32 *)up(DS_A_FLAG, zero, 8);
      target = zone_names_launch(H, d.zone_target, bad);
      const u32 *ub = (const u32 *)up(DS_A_UP + AC_ZONE_REC_B, H.zone_rec_begin, 4 * (size_t)(nz + 1));
      at = (const u32 *)up(DS_A_PAIRS + AT_REC, d.rec_at, 4 * (size_t)ni);
      be.for_each("delta_record_at", nz, FDeltaRecAt{R.zone_rec_begin, target, ub, at, bad + 1});
      u32 flag[2];
      be.download(flag, bad, 8);
      if (flag[0]) return invalid("a delta zone's zone_name differs from the name of the resident zone it targets");
      if (flag[1]) return invalid("rec_at outside the record range of its zone");
    }
    N = R;
    if (ni || nd) {
      stage(H, ni != 0);
      const u32 *ddel = (const u32 *)up(DS_A_DEL + AT_REC, del.data(), 4 * (size_t)nd);
      u32 *src = (u32 *)be.delta_scratch(DS_A_SRC + AT_REC, 4 * (size_t)(n_new + 1));
      if (n + ni) be.for_each("delta_record_map", n + ni, FDeltaZoneMap{ddel, at, nd, ni, n, src});
      const u32 nzones = R.n_zones;
      u32 *zb = (u32 *)standby(AC_ZONE_REC_B, 4 * (size_t)(nzones + 1));
      be.for_each("delta_record_zone_counts", nzones + 1, FDeltaRecZoneCounts{R.zone_rec_begin, ddel, target, U.zone_rec_begin, nd, nz, nzones, zb});
      be.exclusive_scan(zb, nzones + 1);
      const int rc = relayout(AT_REC, src, n_new);
      if (rc != GAR_OK) return rc;
      for (int c = 0; c < AC_N; c++)
        if (written[c]) be.delta_actual_swap(c);
      T.a = N;
    }
    out.n_records = T.a.n_records;
    out.n_values = T.a.n_values;
    out.slab_base = base;
    out.slab_len = T.a.slab_len;
    return GAR_OK;
  }

 private:
  int invalid(const std::string &msg) {
    error = msg;
    return GAR_E_INVALID;
  }
  const void *up(int k, const void *host, size_t bytes) {
    void *p = be.delta_scratch(k, bytes + GAR_SLAB_PAD + 16);
    if (bytes) be.upload(p, host, bytes);
    return p;
  }
  // an empty table: every CSR is {0}
  static gar_actual empty_table() {
    static const u32 kZero[1] = {0};
    gar_actual a{};
    for (int c = 0; c < AC_N; c++)
      if (kActualCols[c].child != AT_N) actual_col(a, c) = kZero;
    return a;
  }
  // the delta rows on the device (U); with append_slab their strings go behind the resident ones at `base`
  void stage(const gar_actual &H, bool append_slab) {
    U = H;
    for (int c = 0; c < AC_N; c++) {
      const ActualColInfo &ci = kActualCols[c];
      const size_t n = (size_t)actual_rows(H, ci.table) + (ci.child != AT_N ? 1 : 0);
      actual_col(U, c) = up(DS_A_UP + c, actual_col(H, c), n * ci.width);
    }
    if (append_slab) {
      u8 *slab = be.delta_actual_slab(R.slab_len, base + H.slab_len + GAR_SLAB_PAD);
      static const u8 kZeros[GAR_SLAB_PAD] = {};
      if (H.slab_len) be.upload(slab + base, H.slab, H.slab_len);
      be.upload(slab + base + H.slab_len, kZeros, GAR_SLAB_PAD);
      T.a.slab = N.slab = slab;  // the resident bytes moved with a grown slab; slab_len changes only with the rest
      N.slab_len = base + H.slab_len;
    }
  }
  void *standby(int c, size_t bytes) {
    written[c] = true;
    void *p = be.delta_actual_col(c, bytes + 16);
    actual_col(N, c) = p;
    return p;
  }

  // targets and deletes of a root table with order-preserving deletes: the compaction keys (deleted rows ascending, minus
  // their rank) and the (new row, source) pairs of the replaced and appended rows
  bool plan(const char *what, u32 n, u32 nu, const u32 *target, u32 nd, const u32 *deleted, std::vector<u32> &key, std::vector<u32> &pairs, u32 &n_new) {
    std::unordered_set<u32> seen;
    for (u32 k = 0; k < nd + nu; k++) {
      const u32 r = k < nd ? deleted[k] : target[k - nd];
      if (k >= nd && r == GAR_NONE) continue;
      if (r >= n) {
        invalid(std::string(what) + " row out of range");
        return false;
      }
      if (!seen.insert(r).second) {
        invalid(std::string("a resident ") + what + " row appears twice among the targets and deleted rows");
        return false;
      }
    }
    key.assign(deleted, deleted + nd);
    std::sort(key.begin(), key.end());
    const u32 survivors = n - nd;
    u32 appended = 0;
    for (u32 k = 0; k < nu; k++) {
      const u32 r = target[k];
      pairs.push_back(r == GAR_NONE ? survivors + appended++ : r - (u32)(std::lower_bound(key.begin(), key.end(), r) - key.begin()));
      pairs.push_back(SRC_UPSERT | k);
    }
    for (u32 m = 0; m < nd; m++) key[m] -= m;
    n_new = survivors + appended;
    return true;
  }

  bool zone_names_match(const gar_actual &H, const u32 *target) {
    const u32 zero = 0;
    u32 *bad = (u32 *)up(DS_A_FLAG, &zero, 4);
    zone_names_launch(H, target, bad);
    u32 flag = 0;
    be.download(&flag, bad, 4);
    return flag == 0;
  }
  // queues the zone-name check (delta zone k against resident zone target[k]; *bad = 1 on a mismatch) -> target on the device
  const u32 *zone_names_launch(const gar_actual &H, const u32 *target, u32 *bad) {
    std::vector<u8> zslab;
    std::vector<gar_str> zref(H.n_zones);
    for (u32 k = 0; k < H.n_zones; k++) {
      const u32 len = GAR_STR_LEN(H.zone_name[k]);
      const u8 *p = H.slab + GAR_STR_OFF(H.zone_name[k]);
      zref[k] = GAR_STR(zslab.size(), len);
      zslab.insert(zslab.end(), p, p + len);
    }
    zslab.resize(zslab.size() + GAR_SLAB_PAD, 0);
    const u32 *dtarget = (const u32 *)up(DS_A_ZTARGET, target, 4 * (size_t)H.n_zones);
    be.for_each("delta_zone_names", H.n_zones,
                FDeltaZoneName{R.slab, R.zone_name, dtarget, (const u8 *)up(DS_A_ZSLAB, zslab.data(), zslab.size()),
                               (const gar_str *)up(DS_A_ZREF, zref.data(), 8 * (size_t)H.n_zones), bad});
    return dtarget;
  }

  // source map of a root table: identity or the survivors of the deletes, then the replaced / appended rows
  const u32 *root_map(int t, u32 n, const std::vector<u32> &key, const std::vector<u32> &pairs) {
    u32 *src = (u32 *)be.delta_scratch(DS_A_SRC + t, 4 * (size_t)(n + 1));
    if (n && key.empty()) be.for_each("delta_source_map", n, FDeltaIdentity{src});
    if (n && !key.empty()) be.for_each("delta_source_map", n, FDeltaCompact{(const u32 *)up(DS_A_DEL + t, key.data(), 4 * key.size()), (u32)key.size(), src});
    if (!pairs.empty()) be.for_each("delta_source_map", (u32)(pairs.size() / 2), FDeltaScatter{(const u32 *)up(DS_A_PAIRS + t, pairs.data(), 4 * pairs.size()), src});
    return src;
  }

  // table t gets the n rows src names: its fixed-width columns are gathered, and each CSR link to a child table yields the new
  // begins (counts + scan) and the children's source map, from which the child table is re-laid in turn
  int relayout(int t, const u32 *src, u32 n) {
    actual_rows(N, t) = n;
    FDeltaGather g{src, base, 0, {}};
    for (int c = 0; c < AC_N; c++) {
      const ActualColInfo &ci = kActualCols[c];
      if (ci.table != t || ci.child != AT_N || (c == AC_ZONE_NAME && !move_zones)) continue;  // an AWS delta keeps every zone row in place
      g.c[g.ncols++] = DeltaGatherCol{(const u8 *)actual_col(R, c), (const u8 *)actual_col(U, c), (u8 *)standby(c, (size_t)n * ci.width), ci.width, ci.str};
    }
    if (g.ncols && n) be.for_each("delta_gather", n, g);
    for (int c = 0; c < AC_N; c++) {
      const ActualColInfo &ci = kActualCols[c];
      if (ci.table != t || ci.child == AT_N) continue;
      const u32 *rb = (const u32 *)actual_col(R, c), *ub = (const u32 *)actual_col(U, c);
      u32 *db = (u32 *)standby(c, 4 * (size_t)(n + 1));
      be.for_each("delta_csr_counts", n + 1, FDeltaCsrCounts{src, rb, ub, n, db});
      be.exclusive_scan(db, n + 1);
      u32 nc = 0;
      be.download(&nc, db + n, 4);
      if (nc >= (1u << 27)) return invalid(std::string(kActualColName[c]) + ": too many rows for one snapshot");
      u32 *csrc = (u32 *)be.delta_scratch(DS_A_SRC + ci.child, 4 * (size_t)(nc + 1));
      if (n) be.for_each("delta_csr_children", n * 32, FDeltaCsrChildren{src, rb, ub, db, csrc});
      const int rc = relayout(ci.child, csrc, nc);
      if (rc != GAR_OK) return rc;
    }
    return GAR_OK;
  }
};
