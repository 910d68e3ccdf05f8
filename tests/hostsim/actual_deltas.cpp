// actual_deltas.cpp — TEST BUILD ONLY: the host simulation with both delta entry points.  This file is the translation unit of
// libgarecon_hostsim.so: it includes deltas.cpp (hostsim.cpp + gar_snapshot_apply_objects) whole and adds
// gar_snapshot_apply_actual, so that the CPU tier runs the AWS-delta splice (ActualSplicer, csrc/gar_delta.h) against the oracle.
// Its buffers are the staging buffers of the engine's DeltaHost (deltas.cpp), which go with the engine.
#include "deltas.cpp"

// the AWS-delta backend of one engine: kernels run on the engine itself, buffers live in its DeltaHost
struct ActualHost {
  gar_engine &e;
  DeltaHost &h;
  template <class F>
  void for_each(const char *name, u32 n, const F &f) { e.for_each(name, n, f); }
  void exclusive_scan(u32 *d, u32 n) { e.exclusive_scan(d, n); }
  void download(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
  void upload(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
  void *delta_scratch(int k, size_t bytes) { return h.scratch[k].ensure(bytes); }
  // column c alternates between two buffers; the standby one is whichever the resident table does not point to (after a load
  // it points to the caller's arrays: either buffer will do)
  void *delta_actual_col(int c, size_t bytes) {
    HBuf &b0 = h.scratch[DS_A_COL + 2 * c];
    HBuf &b = actual_col(e.T.a, c) == (const void *)b0.mem.data() ? h.scratch[DS_A_COL + 2 * c + 1] : b0;
    return b.ensure(bytes);
  }
  void delta_actual_swap(int) {}  // the resident table's pointer is what says which buffer is resident
  u8 *delta_actual_slab(u64, u64 need) {
    std::vector<uint8_t> &s = e.slabs[1];  // gar_snapshot_load copied the AWS slab here
    if (s.size() < need + 16) s.resize(need + need / 2 + 64, 0);  // keeps the resident bytes
    return s.data();
  }
};

extern "C" {

int gar_snapshot_apply_actual(gar_engine *e, const gar_actual_delta *d, gar_actual_delta_result *out) {
  if (!e || !d || !out) return GAR_E_INVALID;
  if (!e->loaded || e->shard_home || e->shard_round != 0) {
    e->err = "no snapshot loaded, or sharded mode";
    return GAR_E_STATE;
  }
  DeltaHost *&h = g_delta[e];
  if (!h) h = new DeltaHost{*e};
  ActualHost be{*e, *h};
  ActualSplicer<ActualHost> S{be, e->T};
  const int rc = S.apply(*d, *out);
  e->slice = e->T;  // the AWS slab may have moved even when the delta was refused (its resident bytes unchanged)
  if (e->pipe) {
    e->pipe->T = e->T;
    if (rc == GAR_OK) e->pipe->prepared = false;  // the next diff prepares the snapshot as the first one after a load
  }
  if (rc != GAR_OK) {
    e->err = S.error;
    return rc;
  }
  return GAR_OK;
}

}  // extern "C"
