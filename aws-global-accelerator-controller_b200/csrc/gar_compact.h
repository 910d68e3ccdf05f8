// gar_compact.h — slab compaction (gar_snapshot_compact): the resident string slabs rebuilt dense on the device.
//
// Shared by the CUDA backend (gar_engine.cu) and the host simulation (tests/hostsim), like gar_delta.h: functors for the
// data-parallel steps plus a driver template, Compactor<B>, that runs them over a Backend.  The layout it produces is the one of
// include/garecon.h "slab compaction": per group, the string columns in struct declaration order, each column's live strings
// back to back.  Because the columns follow each other without padding, the strings of a group form ONE sequence (column 0's
// rows, column 1's rows, ...) and the steps run on that concatenation, not per column:
//   1. lengths: one fused launch over all columns writes, per string, its normalised source reference (the object key is one
//      "ns/name" string; a row whose flag says "no value" is empty and its reference is never read) and its live length;
//   2. offsets: ONE 64-bit exclusive scan over the concatenated lengths gives every string's offset in the new slab and, as
//      its last element, the new slab_len (offsets are 40-bit: a u32 scan would wrap);
//   3. copy (Backend::compact_copy): the new slab is cut into windows of COMPACT_WINDOW destination bytes; a window finds its
//      first string by binary search in the offsets and copies what falls inside it.  Old and new slab are distinct buffers;
//   4. rewrite: one fused launch writes the gar_str columns into standby buffers; then the standby buffers and the new slab
//      become resident and the old slab is freed.
// Nothing resident changes before step 4 has been queued for every selected group.
//
// The export (gar_snapshot_export, Compactor::export_to) runs steps 1 and 2 unchanged and steps 3 and 4 with a destination
// outside the resident set: the rewrite writes into export staging, the copy gathers the new slab chunk by chunk into a small
// ring of device slots that a second stream copies into the caller's host buffer, and nothing is committed.
//
// Backend interface, on top of gar_delta.h's:
//   void exclusive_scan(u64 *data, u32 n);
//   u8 *compact_slab(int g, u64 bytes);        // a fresh buffer for group g's new slab; nullptr: out of memory
//   void compact_slab_commit(int g, bool keep); // keep: the fresh buffer replaces group g's resident slab, which is freed;
//                                               // otherwise the fresh buffer is freed
//   void compact_copy(u8 *dst, const u8 *src, const gar_str *sref, const u64 *off, u32 m, u64 total, bool any_long);
// and for the export only:
//   void *export_stage(int g, size_t bytes);   // device staging of group g's rewritten gar_str columns; nullptr: out of memory
//   void *export_scratch(int k, size_t bytes); // the per-string staging (CS_*) of an export; nullptr: out of memory
//   void export_fence();                       // later export copies wait for the work queued on the main stream so far
//   void export_copy(void *host, const void *dev, size_t bytes);  // device -> caller's buffer, behind the last export_fence
//   int export_slab(u8 *host, const u8 *src, const gar_str *sref, const u64 *off, u32 m, u64 total, bool any_long);
//                                              // step 3 into the caller's buffer; GAR_E_NOMEM: no ring
#pragma once

#include "gar_delta.h"

constexpr u32 COMPACT_WINDOW = 32 * 1024;  // destination bytes per window (one block on the GPU); a multiple of 16
constexpr u32 COMPACT_LONG = 1024;         // longer strings are copied by the long-string launch, spread over whole blocks
enum { CG_OBJECTS = 0, CG_ACTUAL = 1, CG_N = 2 };
// the export gathers the new slab EXPORT_CHUNK windows (4 MiB) at a time into a ring of EXPORT_RING slots
constexpr u32 EXPORT_CHUNK = 128;
constexpr int EXPORT_RING = 4;
// a compaction and a delta never run at the same time: the staging buffers are the deltas' (group g uses CS_x + g)
enum CompactScratch { CS_SREF = DS_KEY_REF, CS_OFF = DS_OFFS, CS_HEAD = DS_TOTALS };
static_assert(DS_KEY_SLAB == DS_KEY_REF + 1 && DS_ROWS == DS_OFFS + 1, "two consecutive staging buffers per kind");

// one string column of a group
struct CompactCol {
  const gar_str *ref;   // resident column (the key column: obj_ns)
  const gar_str *name;  // the key column: obj_name (the key is len(ns) + 1 + len(name) bytes from obj_ns's offset); else nullptr
  const u8 *gate;       // rows with (gate[i] & mask) == 0 count as empty and their reference is not read; nullptr: every row is live
  gar_str *out, *out_name;  // standby columns
  u32 n, pos;           // rows; position of row 0 in the concatenated sequence
  u8 mask;
};
struct FCompactLen {
  CompactCol c;
  gar_str *sref;
  u64 *len;
  u32 *any_long;
  GAR_HD void operator()(u32 i) const {
    gar_str r = 0;
    if (!c.gate || (c.gate[i] & c.mask)) {
      r = c.ref[i];
      if (c.name) r = GAR_STR(GAR_STR_OFF(r), GAR_STR_LEN(r) + 1 + GAR_STR_LEN(c.name[i]));
    }
    sref[c.pos + i] = r;
    len[c.pos + i] = GAR_STR_LEN(r);
    if (GAR_STR_LEN(r) > COMPACT_LONG) *any_long = 1;
  }
};
// head words of a group: [0] any string longer than COMPACT_LONG, [2..3] the new slab_len
struct FCompactHead {
  const u64 *total;
  u32 *head;
  GAR_HD void operator()(u32) const {
    head[2] = (u32)*total;
    head[3] = (u32)(*total >> 32);
  }
};
struct FCompactRewrite {
  CompactCol c;
  const gar_str *sref;
  const u64 *off;
  GAR_HD void operator()(u32 i) const {
    const u64 o = off[c.pos + i];
    if (c.name) {  // both halves of the key reference the one copy
      const u32 ln = GAR_STR_LEN(c.ref[i]);
      c.out[i] = GAR_STR(o, ln);
      c.out_name[i] = GAR_STR(o + ln + 1, GAR_STR_LEN(c.name[i]));
    } else {
      c.out[i] = GAR_STR(o, GAR_STR_LEN(sref[c.pos + i]));
    }
  }
};

// the strings that overlap destination bytes [lo, hi): positions [compact_first(lo), compact_end(hi)) of the sequence.
// off[0 .. m] ascending, off[m] = total; empty strings that sit exactly at lo are skipped (nothing of them is in the window)
GAR_HD u32 compact_first(const u64 *off, u32 m, u64 lo) {  // the last position with off[p] <= lo
  u32 a = 0, b = m + 1;
  while (b - a > 1) {
    const u32 mid = a + ((b - a) >> 1);
    if (off[mid] <= lo) a = mid;
    else b = mid;
  }
  return a;
}
GAR_HD u32 compact_end(const u64 *off, u32 m, u64 hi) {  // the first position with off[p] >= hi
  u32 a = 0, b = m;
  while (a < b) {
    const u32 mid = a + ((b - a) >> 1);
    if (off[mid] < hi) a = mid + 1;
    else b = mid;
  }
  return a;
}
// window w0 + w copied serially: the form a backend without shared memory runs (the host simulation).  dst holds the windows
// from w0 on (dst[0] is destination byte w0 * COMPACT_WINDOW)
struct FCompactWindow {
  u8 *dst;
  const u8 *src;
  const gar_str *sref;
  const u64 *off;
  u32 m;
  u64 total;
  u32 w0 = 0;
  GAR_HD void operator()(u32 w) const {
    const u64 base = (u64)w0 * COMPACT_WINDOW, lo = base + (u64)w * COMPACT_WINDOW, hi = lo + COMPACT_WINDOW < total ? lo + COMPACT_WINDOW : total;
    const u32 p0 = compact_first(off, m, lo), p1 = compact_end(off, m, hi);
    for (u32 p = p0; p < p1; p++) {
      const u64 o = off[p], e = o + GAR_STR_LEN(sref[p]);
      const u64 a = o > lo ? o : lo, b = e < hi ? e : hi;
      const u8 *s = src + GAR_STR_OFF(sref[p]);
      for (u64 k = a; k < b; k++) dst[k - base] = s[k - o];
    }
  }
};

// one column of a group as gar_snapshot_export lays it out in the caller's buffer: the struct field of its pointer, the field of
// its row count, element width, gar_str or not, CSR (n + 1 entries) or not
struct ExportColInfo {
  size_t field, rows;
  u8 width, str, csr;
};
#define GAR_OC(f, r, w, s, c) ExportColInfo{offsetof(gar_objects, f), offsetof(gar_objects, r), w, s, c}
static const ExportColInfo kObjectCols[DC_N] = {  // gar_objects order = DC_* order
    GAR_OC(obj_kind, n_objects, 1, 0, 0),      GAR_OC(obj_spec_type, n_objects, 1, 0, 0), GAR_OC(obj_flags, n_objects, 1, 0, 0),
    GAR_OC(obj_ns, n_objects, 8, 1, 0),        GAR_OC(obj_name, n_objects, 8, 1, 0),      GAR_OC(obj_ingress_class, n_objects, 8, 1, 0),
    GAR_OC(obj_ann_begin, n_objects, 4, 0, 1), GAR_OC(obj_lbi_begin, n_objects, 4, 0, 1), GAR_OC(obj_port_begin, n_objects, 4, 0, 1),
    GAR_OC(ann_key, n_ann, 8, 1, 0),           GAR_OC(ann_val, n_ann, 8, 1, 0),           GAR_OC(lbi_hostname, n_lbi, 8, 1, 0),
    GAR_OC(port_number, n_ports, 4, 0, 0),     GAR_OC(port_proto, n_ports, 8, 1, 0)};
#undef GAR_OC

template <class B>
struct Compactor {
  B &be;
  DevTables &T;  // the resident tables: the string columns and slabs of the selected groups are replaced
  std::string error;
  Compactor(B &be_, DevTables &T_) : be(be_), T(T_) {}

  // GAR_OK; GAR_E_NOMEM or GAR_E_INVALID (error says why): nothing resident changed
  int run(u32 groups, gar_compact_result &out) {
    out.obj_slab_before = out.obj_slab_len = T.o.slab_len;
    out.act_slab_before = out.act_slab_len = T.a.slab_len;
    Group G[CG_N];
    if (groups & GAR_COMPACT_OBJECTS) plan_objects(G[CG_OBJECTS], nullptr);
    if (groups & GAR_COMPACT_ACTUAL) plan_actual(G[CG_ACTUAL], nullptr);
    int rc = GAR_OK;
    for (int g = 0; g < CG_N && rc == GAR_OK; g++) {
      if (!G[g].ncols) continue;
      G[g].sref = (gar_str *)be.delta_scratch(CS_SREF + g, scratch_bytes(G[g]));
      G[g].off = (u64 *)be.delta_scratch(CS_OFF + g, scratch_bytes(G[g]));
      rc = measure(g, G[g]);
      if (rc == GAR_OK && !(G[g].slab = be.compact_slab(g, G[g].total + GAR_SLAB_PAD + 16))) {
        error = "out of device memory for the compacted slab";
        rc = GAR_E_NOMEM;
      }
    }
    if (rc != GAR_OK) {
      for (int g = 0; g < CG_N; g++)
        if (G[g].slab) be.compact_slab_commit(g, false);
      return rc;
    }
    for (int g = 0; g < CG_N; g++)
      if (G[g].ncols) copy_and_rewrite(g, G[g]);
    if (G[CG_OBJECTS].ncols) {
      be.delta_swap();
      be.compact_slab_commit(CG_OBJECTS, true);
      T.o = No;
      out.obj_slab_len = T.o.slab_len;
    }
    if (G[CG_ACTUAL].ncols) {
      for (int c = 0; c < AC_N; c++)
        if (kActualCols[c].str) be.delta_actual_swap(c);
      be.compact_slab_commit(CG_ACTUAL, true);
      T.a = Na;
      out.act_slab_len = T.a.slab_len;
    }
    return GAR_OK;
  }

  // gar_snapshot_export: steps 1 and 2 as above, then the rewrite into export staging and the copy into the caller's host buffer
  // buf[g] (cap[g] bytes; nullptr: a size query for group g, nothing is written).  Columns in struct order, each at a 16-byte
  // aligned offset, the slab last; *obj_out / *act_out point into the buffers.  Nothing resident changes.
  // GAR_OK; GAR_E_INVALID (a buffer too small; out holds the bytes needed) or GAR_E_NOMEM (error says why)
  int export_to(u32 groups, u8 *const buf[CG_N], const u64 cap[CG_N], gar_objects *obj_out, gar_actual *act_out, gar_export_result &out) {
    out = gar_export_result{};
    Group G[CG_N];
    Export X[CG_N];
    if (groups & GAR_COMPACT_OBJECTS) {
      layout(X[CG_OBJECTS], &T.o, kObjectCols, DC_N);
      if (!stage(CG_OBJECTS, X[CG_OBJECTS], buf[CG_OBJECTS])) return GAR_E_NOMEM;
      plan_objects(G[CG_OBJECTS], &X[CG_OBJECTS]);
    }
    if (groups & GAR_COMPACT_ACTUAL) {
      ExportColInfo ac[AC_N];
      for (int c = 0; c < AC_N; c++) {
        const ActualColInfo &ci = kActualCols[c];
        ac[c] = ExportColInfo{ci.field, kActualRows[ci.table], ci.width, ci.str, (u8)(ci.child != AT_N)};
      }
      layout(X[CG_ACTUAL], &T.a, ac, AC_N);
      if (!stage(CG_ACTUAL, X[CG_ACTUAL], buf[CG_ACTUAL])) return GAR_E_NOMEM;
      plan_actual(G[CG_ACTUAL], &X[CG_ACTUAL]);
    }
    // the fixed-width columns and CSRs travel straight from the resident buffers while the lengths pass runs
    be.export_fence();
    for (int g = 0; g < CG_N; g++)
      if (G[g].ncols && buf[g] && X[g].slab_at <= cap[g])
        for (int c = 0; c < X[g].ncols; c++)
          if (!X[g].col[c].str) be.export_copy(buf[g] + X[g].col[c].at, X[g].col[c].src, X[g].col[c].bytes);
    bool fits = true;
    for (int g = 0; g < CG_N; g++) {
      if (!G[g].ncols) continue;
      G[g].sref = (gar_str *)be.export_scratch(CS_SREF + g, scratch_bytes(G[g]));
      G[g].off = (u64 *)be.export_scratch(CS_OFF + g, scratch_bytes(G[g]));
      if (!G[g].sref || !G[g].off) {
        error = "out of device memory for the per-string staging of the export";
        return GAR_E_NOMEM;
      }
      if (const int rc = measure(g, G[g])) return rc;
      const u64 need = X[g].slab_at + G[g].total;
      (g == CG_OBJECTS ? out.obj_bytes : out.act_bytes) = need;
      (g == CG_OBJECTS ? out.obj_slab_len : out.act_slab_len) = G[g].total;
      if (buf[g] && need > cap[g]) fits = false;
    }
    if (!fits) {
      error = "the buffer is smaller than the exported tables (the bytes needed are in the result)";
      return GAR_E_INVALID;
    }
    for (int g = 0; g < CG_N; g++) {
      if (!G[g].ncols || !buf[g]) continue;
      FCompactRewrite fr[AC_N];
      for (int k = 0; k < G[g].ncols; k++) fr[k] = FCompactRewrite{G[g].col[k], G[g].sref, G[g].off};
      fused("compact_rewrite", G[g], fr);
      be.export_fence();
      for (int c = 0; c < X[g].ncols; c++)
        if (X[g].col[c].str) be.export_copy(buf[g] + X[g].col[c].at, X[g].stage + X[g].col[c].stage_at, X[g].col[c].bytes);
      if (be.export_slab(buf[g] + X[g].slab_at, G[g].old_slab, G[g].sref, G[g].off, G[g].m, G[g].total, G[g].any_long) != GAR_OK) {
        error = "out of device memory for the export ring";
        return GAR_E_NOMEM;
      }
    }
    if (buf[CG_OBJECTS] && G[CG_OBJECTS].ncols) finish(X[CG_OBJECTS], T.o, *obj_out, buf[CG_OBJECTS], G[CG_OBJECTS].total);
    if (buf[CG_ACTUAL] && G[CG_ACTUAL].ncols) finish(X[CG_ACTUAL], T.a, *act_out, buf[CG_ACTUAL], G[CG_ACTUAL].total);
    return GAR_OK;
  }

 private:
  struct Group {
    CompactCol col[AC_N];
    int ncols = 0;
    u32 m = 0;  // strings of the group
    const u8 *old_slab = nullptr;
    u8 *slab = nullptr;
    gar_str *sref = nullptr;
    u64 *off = nullptr;
    u64 total = 0;
    bool any_long = false;
  };
  gar_objects No{};
  gar_actual Na{};
  // an export's columns of one group: where each goes in the caller's buffer and, for a gar_str column, its staging on the device
  struct Export {
    struct Col {
      size_t field;
      const void *src;    // resident column
      u64 bytes, at;      // at: offset in the caller's buffer (16-byte aligned)
      u64 stage_at;       // a gar_str column: offset of its rewritten copy in the staging buffer
      bool str;
    } col[AC_N];
    int ncols = 0;
    u64 slab_at = 0, stage_bytes = 0;
    u8 *stage = nullptr;  // the staging buffer; nullptr in a size query, which rewrites nothing
  };
  template <class Tab>
  static void layout(Export &X, const Tab *t, const ExportColInfo *info, int n) {
    u64 at = 0;
    for (int c = 0; c < n; c++) {
      const ExportColInfo &ci = info[c];
      const u64 rows = *(const u32 *)((const char *)t + ci.rows) + (u64)ci.csr;
      auto &x = X.col[X.ncols++];
      x = {ci.field, *(const void *const *)((const char *)t + ci.field), rows * ci.width, at, X.stage_bytes, ci.str != 0};
      at = (at + x.bytes + 15) & ~(u64)15;
      if (x.str) X.stage_bytes = (X.stage_bytes + x.bytes + 15) & ~(u64)15;
    }
    X.slab_at = at;
  }
  // the staging buffer of the rewritten gar_str columns (a size query rewrites nothing and needs none)
  bool stage(int g, Export &X, const u8 *buf) {
    if (!buf) return true;
    X.stage = (u8 *)be.export_stage(g, X.stage_bytes + 16);
    if (!X.stage) {
      error = "out of device memory for the export staging";
      return false;
    }
    return true;
  }
  // where the rewrite writes gar_str column `field` (nullptr in a size query)
  static gar_str *staged(const Export &X, size_t field) {
    if (X.stage)
      for (int c = 0; c < X.ncols; c++)
        if (X.col[c].field == field) return (gar_str *)(X.stage + X.col[c].stage_at);
    return nullptr;
  }
  template <class Tab>
  static void finish(const Export &X, const Tab &resident, Tab &out, u8 *buf, u64 total) {
    out = resident;
    for (int c = 0; c < X.ncols; c++) *(const void **)((char *)&out + X.col[c].field) = buf + X.col[c].at;
    out.slab = buf + X.slab_at;
    out.slab_len = total;
  }

  static void add(Group &G, const gar_str *ref, gar_str *out, u32 n, const gar_str *name = nullptr, gar_str *out_name = nullptr, const u8 *gate = nullptr,
                  u8 mask = 0) {
    G.col[G.ncols++] = CompactCol{ref, name, gate, out, out_name, n, G.m, mask};
    G.m += n;
  }
  template <class Tp>
  Tp *standby(int c, const Tp *resident, size_t count, bool copy) {
    Tp *p = (Tp *)be.delta_col(c, count * sizeof(Tp) + 16);
    if (copy) be.copy_bytes(p, resident, count * sizeof(Tp));
    return p;
  }
  // the whole object column set alternates (gar_delta.h): the fixed-width columns and CSRs move to the standby set unchanged.
  // X: an export; the rewritten gar_str columns go to its staging and no standby buffer is touched
  void plan_objects(Group &G, Export *X) {
    const gar_objects &O = T.o;
    const u32 n = O.n_objects;
    auto out = [&](int c, const gar_str *resident, size_t count, size_t field) { return X ? staged(*X, field) : standby(c, resident, count, false); };
    if (!X) {
      No = O;
      No.obj_kind = standby(DC_KIND, O.obj_kind, n, true);
      No.obj_spec_type = standby(DC_SPEC, O.obj_spec_type, n, true);
      No.obj_flags = standby(DC_FLAGS, O.obj_flags, n, true);
      No.obj_ann_begin = standby(DC_ANN_B, O.obj_ann_begin, (size_t)n + 1, true);
      No.obj_lbi_begin = standby(DC_LBI_B, O.obj_lbi_begin, (size_t)n + 1, true);
      No.obj_port_begin = standby(DC_PORT_B, O.obj_port_begin, (size_t)n + 1, true);
      No.port_number = standby(DC_PORT_NUM, O.port_number, O.n_ports, true);
    }
    gar_str *ns = out(DC_NS, O.obj_ns, n, offsetof(gar_objects, obj_ns)), *name = out(DC_NAME, O.obj_name, n, offsetof(gar_objects, obj_name));
    gar_str *icls = out(DC_ICLS, O.obj_ingress_class, n, offsetof(gar_objects, obj_ingress_class));
    gar_str *ann_key = out(DC_ANN_KEY, O.ann_key, O.n_ann, offsetof(gar_objects, ann_key)), *ann_val = out(DC_ANN_VAL, O.ann_val, O.n_ann, offsetof(gar_objects, ann_val));
    gar_str *lbi = out(DC_LBI_HOST, O.lbi_hostname, O.n_lbi, offsetof(gar_objects, lbi_hostname));
    gar_str *proto = out(DC_PORT_PROTO, O.port_proto, O.n_ports, offsetof(gar_objects, port_proto));
    add(G, O.obj_ns, ns, n, O.obj_name, name);
    add(G, O.obj_ingress_class, icls, n, nullptr, nullptr, O.obj_flags, GAR_OBJ_HAS_INGRESS_CLASS);
    add(G, O.ann_key, ann_key, O.n_ann);
    add(G, O.ann_val, ann_val, O.n_ann);
    add(G, O.lbi_hostname, lbi, O.n_lbi);
    add(G, O.port_proto, proto, O.n_ports);
    if (!X) {
      No.obj_ns = ns;
      No.obj_name = name;
      No.obj_ingress_class = icls;
      No.ann_key = ann_key;
      No.ann_val = ann_val;
      No.lbi_hostname = lbi;
      No.port_proto = proto;
    }
    G.old_slab = O.slab;
  }
  void plan_actual(Group &G, Export *X) {
    if (!X) Na = T.a;
    for (int c = 0; c < AC_N; c++) {
      const ActualColInfo &ci = kActualCols[c];
      if (!ci.str) continue;
      const u32 n = actual_rows(T.a, ci.table);
      gar_str *out = X ? staged(*X, ci.field) : (gar_str *)be.delta_actual_col(c, 8 * (size_t)n + 16);
      if (c == AC_REC_ALIAS_DNS) add(G, T.a.rec_alias_dns, out, n, nullptr, nullptr, T.a.rec_has_alias, 0xFF);
      else add(G, (const gar_str *)actual_col(T.a, c), out, n);
      if (!X) actual_col(Na, c) = out;
    }
    G.old_slab = T.a.slab;
  }

  // one launch per MULTI_MAX (8) columns: the object group's six columns in one, the AWS group's thirteen in two
  template <class F>
  void fused(const char *name, const Group &G, const F *f) {
    for (int k = 0; k < G.ncols; k += 8) {
      F g[8];
      u32 n[8] = {};
      for (int j = 0; j < 8; j++) {
        g[j] = f[k + j < G.ncols ? k + j : k];
        if (k + j < G.ncols) n[j] = G.col[k + j].n;
      }
      be.for_each_multi(name, {n[0], n[1], n[2], n[3], n[4], n[5], n[6], n[7]}, g[0], g[1], g[2], g[3], g[4], g[5], g[6], g[7]);
    }
  }

  static size_t scratch_bytes(const Group &G) { return 8 * (size_t)(G.m + 1) + 16; }
  // steps 1 and 2 into G.sref and G.off (scratch_bytes each)
  int measure(int g, Group &G) {
    const u32 m = G.m;
    u32 *head = (u32 *)be.delta_scratch(CS_HEAD, 64) + 4 * g;
    be.fill32((u32 *)(G.off + m), 0, 2);
    be.fill32(head, 0, 4);
    FCompactLen fl[AC_N];
    for (int k = 0; k < G.ncols; k++) fl[k] = FCompactLen{G.col[k], G.sref, G.off, head};
    fused("compact_lengths", G, fl);
    be.exclusive_scan(G.off, m + 1);
    be.for_each("compact_lengths", 1, FCompactHead{G.off + m, head});
    u32 h[4];
    be.download(h, head, sizeof(h));
    G.any_long = h[0] != 0;
    G.total = (u64)h[2] | ((u64)h[3] << 32);
    if (G.total + GAR_SLAB_PAD >= (1ull << GAR_STR_OFF_BITS)) {
      error = "the compacted slab would outgrow 2^40 bytes (strings that shared bytes are copied once per reference)";
      return GAR_E_INVALID;
    }
    return GAR_OK;
  }
  // steps 3 and 4
  void copy_and_rewrite(int g, Group &G) {
    static const u8 kZeros[GAR_SLAB_PAD] = {};
    be.compact_copy(G.slab, G.old_slab, G.sref, G.off, G.m, G.total, G.any_long);
    be.upload(G.slab + G.total, kZeros, GAR_SLAB_PAD);
    FCompactRewrite fr[AC_N];
    for (int k = 0; k < G.ncols; k++) fr[k] = FCompactRewrite{G.col[k], G.sref, G.off};
    fused("compact_rewrite", G, fr);
    if (g == CG_OBJECTS) {
      No.slab = G.slab;
      No.slab_len = G.total;
    } else {
      Na.slab = G.slab;
      Na.slab_len = G.total;
    }
  }
};
