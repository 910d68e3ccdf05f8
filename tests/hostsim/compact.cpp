// compact.cpp — TEST BUILD ONLY: the host simulation with the delta entry points and slab compaction.  This file is the
// translation unit of libgarecon_hostsim.so: it includes actual_deltas.cpp (hostsim.cpp + both delta entry points) whole and adds
// gar_snapshot_compact and gar_snapshot_read_slab, so that the CPU tier runs the compaction driver (Compactor, csrc/gar_compact.h)
// and its window logic against the numpy statement of the layout.  Its buffers are those of the engine's DeltaHost (deltas.cpp).
#include "actual_deltas.cpp"

#include "../../aws-global-accelerator-controller_b200/csrc/gar_compact.h"

// the compaction backend of one engine: kernels run on the engine itself, columns and staging buffers live in its DeltaHost
struct CompactHost {
  gar_engine &e;
  DeltaHost &h;
  ActualHost a;
  std::vector<uint8_t> fresh[CG_N];
  template <class F>
  void for_each(const char *name, u32 n, const F &f) { e.for_each(name, n, f); }
  template <class... Fs>
  void for_each_multi(const char *name, std::initializer_list<u32> ns, const Fs &...fs) { e.for_each_multi(name, ns, fs...); }
  void fill32(u32 *p, u32 v, size_t n) { e.fill32(p, v, n); }
  void exclusive_scan(u64 *d, u32 n) {
    u64 run = 0;
    for (u32 i = 0; i < n; i++) {
      const u64 v = d[i];
      d[i] = run;
      run += v;
    }
  }
  void download(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
  void upload(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
  void copy_bytes(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
  void *delta_scratch(int k, size_t bytes) { return h.delta_scratch(k, bytes); }
  void *delta_col(int c, size_t bytes) { return h.delta_col(c, bytes); }
  void delta_swap() { h.delta_swap(); }
  void *delta_actual_col(int c, size_t bytes) { return a.delta_actual_col(c, bytes); }
  void delta_actual_swap(int c) { a.delta_actual_swap(c); }
  // exactly `bytes` long: a read or write outside the new slab is outside the allocation
  u8 *compact_slab(int g, u64 bytes) {
    fresh[g].assign(bytes, 0xEE);
    return fresh[g].data();
  }
  void compact_slab_commit(int g, bool keep) {
    if (keep) e.slabs[g].swap(fresh[g]);
    std::vector<uint8_t>().swap(fresh[g]);
  }
  void compact_copy(u8 *dst, const u8 *src, const gar_str *sref, const u64 *off, u32 m, u64 total, bool) {
    e.for_each("compact_copy", (u32)((total + COMPACT_WINDOW - 1) / COMPACT_WINDOW), FCompactWindow{dst, src, sref, off, m, total});
  }
};

extern "C" {

int gar_snapshot_compact(gar_engine *e, uint32_t groups, gar_compact_result *out) {
  if (!e || !out) return GAR_E_INVALID;
  if (!groups || (groups & ~(u32)(GAR_COMPACT_OBJECTS | GAR_COMPACT_ACTUAL))) {
    e->err = "groups must be a non-empty mask of GAR_COMPACT_OBJECTS | GAR_COMPACT_ACTUAL";
    return GAR_E_INVALID;
  }
  if (!e->loaded || e->shard_home || e->shard_round != 0) {
    e->err = "no snapshot loaded, or sharded mode";
    return GAR_E_STATE;
  }
  DeltaHost *&h = g_delta[e];
  if (!h) h = new DeltaHost{*e};
  CompactHost be{*e, *h, ActualHost{*e, *h}, {}};
  Compactor<CompactHost> C(be, e->T);
  const int rc = C.run(groups, *out);
  if (rc != GAR_OK) {
    e->err = C.error;
    return rc;
  }
  e->slice = e->T;
  if (e->pipe) {
    e->pipe->T = e->T;
    if (groups & GAR_COMPACT_OBJECTS) e->pipe->obj_stale = true;
    if (groups & GAR_COMPACT_ACTUAL) e->pipe->prepared = false;
  }
  return GAR_OK;
}

int gar_snapshot_read_slab(gar_engine *e, uint32_t group, uint64_t off, uint64_t len, void *dst) {
  if (!e) return GAR_E_INVALID;
  if (group != GAR_COMPACT_OBJECTS && group != GAR_COMPACT_ACTUAL) {
    e->err = "group must be GAR_COMPACT_OBJECTS or GAR_COMPACT_ACTUAL";
    return GAR_E_INVALID;
  }
  if (!e->loaded || e->shard_home) {
    e->err = "no snapshot loaded, or a sharded sub-snapshot";
    return GAR_E_STATE;
  }
  const u8 *slab = group == GAR_COMPACT_OBJECTS ? e->T.o.slab : e->T.a.slab;
  const u64 slab_len = group == GAR_COMPACT_OBJECTS ? e->T.o.slab_len : e->T.a.slab_len;
  if (off > slab_len || len > slab_len - off || (len && !dst)) {
    e->err = "off + len beyond the resident slab_len";
    return GAR_E_INVALID;
  }
  if (len) memcpy(dst, slab + off, len);
  return GAR_OK;
}

}  // extern "C"
