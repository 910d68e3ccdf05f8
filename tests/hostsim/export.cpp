// export.cpp — TEST BUILD ONLY: the host simulation with every delta entry point, slab compaction, zone deltas and the export.
// This file is the translation unit of libgarecon_hostsim.so: it includes zone_deltas.cpp (hostsim.cpp + the object, AWS and
// zone deltas + the compaction) whole and adds gar_snapshot_export, so that the CPU tier runs the export driver
// (Compactor::export_to, csrc/gar_compact.h) against the numpy statement of the layout.  The slab is gathered as on the GPU:
// EXPORT_CHUNK windows at a time (the serial window copy over a window range) into a ring slot, then into the caller's buffer.
#include "zone_deltas.cpp"

// the export backend: the compaction's, plus staging that is plain host memory and copies that are memcpy
struct ExportHost : CompactHost {
  std::vector<uint8_t> stage[CG_N];
  void *export_stage(int g, size_t bytes) {
    stage[g].assign(bytes, 0xEE);
    return stage[g].data();
  }
  void *export_scratch(int k, size_t bytes) { return h.delta_scratch(k, bytes); }
  void export_fence() {}
  void export_copy(void *host, const void *dev, size_t bytes) { memcpy(host, dev, bytes); }
  int export_slab(u8 *host, const u8 *src, const gar_str *sref, const u64 *off, u32 m, u64 total, bool) {
    const u32 windows = (u32)((total + COMPACT_WINDOW - 1) / COMPACT_WINDOW);
    std::vector<uint8_t> ring[EXPORT_RING];
    for (u32 w0 = 0, k = 0; w0 < windows; w0 += EXPORT_CHUNK, k++) {
      std::vector<uint8_t> &slot = ring[k % EXPORT_RING];
      const u64 lo = (u64)w0 * COMPACT_WINDOW, bytes = std::min<u64>((u64)EXPORT_CHUNK * COMPACT_WINDOW, total - lo);
      slot.assign(bytes, 0xEE);  // exactly the chunk: a write outside it is outside the allocation
      e.for_each("compact_copy", std::min(EXPORT_CHUNK, windows - w0), FCompactWindow{slot.data(), src, sref, off, m, total, w0});
      memcpy(host + lo, slot.data(), bytes);
    }
    return GAR_OK;
  }
};

extern "C" {

int gar_snapshot_export(gar_engine *e, uint32_t groups, void *obj_buf, uint64_t obj_cap, gar_objects *obj_out, void *act_buf, uint64_t act_cap,
                        gar_actual *act_out, gar_export_result *out) {
  if (!e || !out) return GAR_E_INVALID;
  if (!groups || (groups & ~(u32)(GAR_COMPACT_OBJECTS | GAR_COMPACT_ACTUAL)) || ((groups & GAR_COMPACT_OBJECTS) && !obj_out) ||
      ((groups & GAR_COMPACT_ACTUAL) && !act_out)) {
    e->err = "groups must be a non-empty mask of GAR_COMPACT_OBJECTS | GAR_COMPACT_ACTUAL, with a table struct for each";
    return GAR_E_INVALID;
  }
  if (!e->loaded || e->shard_home || e->shard_round != 0) {
    e->err = "no snapshot loaded, or sharded mode";
    return GAR_E_STATE;
  }
  DeltaHost *&h = g_delta[e];
  if (!h) h = new DeltaHost{*e};
  ExportHost be{{*e, *h, ActualHost{*e, *h}, {}}, {}};
  u8 *const buf[CG_N] = {(groups & GAR_COMPACT_OBJECTS) ? (u8 *)obj_buf : nullptr, (groups & GAR_COMPACT_ACTUAL) ? (u8 *)act_buf : nullptr};
  const u64 cap[CG_N] = {obj_cap, act_cap};
  Compactor<ExportHost> C(be, e->T);
  const int rc = C.export_to(groups, buf, cap, obj_out, act_out, *out);
  if (rc != GAR_OK) {
    e->err = C.error;
    return rc;
  }
  return GAR_OK;
}

}  // extern "C"
