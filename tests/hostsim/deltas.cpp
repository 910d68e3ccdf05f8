// deltas.cpp — TEST BUILD ONLY: the host simulation (hostsim.cpp) plus gar_snapshot_apply_objects, so that the CPU tier runs
// the object-delta splice (csrc/gar_delta.h) against the oracle.  This file is the translation unit of
// libgarecon_hostsim.so: it includes hostsim.cpp whole and adds, beside its backend, the buffers a splice writes — the two
// alternating object column sets and the staging buffers.  hostsim.cpp's destroy entry point is wrapped so that they go with
// the engine.
#include <unordered_map>

#define gar_engine_destroy hostsim_engine_destroy
#include "hostsim.cpp"
#undef gar_engine_destroy

#include "../../aws-global-accelerator-controller_b200/csrc/gar_delta.h"

// the delta buffers of one engine; its pipeline keeps running on the engine itself (hostsim.cpp's backend)
struct DeltaHost {
  gar_engine &e;
  HBuf col[2][DC_N], scratch[DS_N];
  int o_set = -1;  // col[o_set] is resident unless a load replaced it by the caller's arrays: a splice always writes the other set
  template <class F>
  void for_each(const char *name, u32 n, const F &f) { e.for_each(name, n, f); }
  void exclusive_scan(u32 *d, u32 n) { e.exclusive_scan(d, n); }
  void download(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
  void upload(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
  void *delta_scratch(int k, size_t bytes) { return scratch[k].ensure(bytes); }
  void *delta_col(int c, size_t bytes) { return col[o_set == 0 ? 1 : 0][c].ensure(bytes); }
  void delta_swap() { o_set = o_set == 0 ? 1 : 0; }
  u8 *delta_slab(u64, u64 need) {
    std::vector<uint8_t> &s = e.slabs[0];  // gar_snapshot_load copied the object slab here
    if (s.size() < need + 16) s.resize(need + need / 2 + 64, 0);  // keeps the resident bytes
    return s.data();
  }
};
static std::unordered_map<gar_engine *, DeltaHost *> g_delta;

extern "C" {

void gar_engine_destroy(gar_engine *e) {
  auto it = g_delta.find(e);
  if (it != g_delta.end()) {
    delete it->second;
    g_delta.erase(it);
  }
  hostsim_engine_destroy(e);
}

int gar_snapshot_apply_objects(gar_engine *e, const gar_object_delta *d, gar_delta_result *out) {
  if (!e || !d || !out) return GAR_E_INVALID;
  if (!e->loaded || e->shard_home || e->shard_round != 0) {
    e->err = "no snapshot loaded, or sharded mode";
    return GAR_E_STATE;
  }
  if (!e->pipe) {  // as diff_impl creates it
    e->pipe = new Pipeline<gar_engine>(*e, e->T);
    if (const char *tc = getenv("GAR_TINY_CAPS")) e->pipe->tiny_caps = tc[0] == '1';
  }
  DeltaHost *&h = g_delta[e];
  if (!h) h = new DeltaHost{*e};
  Splicer<DeltaHost, gar_engine> S{*h, *e->pipe, e->T};
  const int rc = S.apply(*d, *out);
  if (rc != GAR_OK) {
    e->err = S.error;
    return rc;
  }
  e->slice = e->T;
  return GAR_OK;
}

}  // extern "C"
