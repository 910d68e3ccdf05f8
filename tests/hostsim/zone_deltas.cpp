// zone_deltas.cpp — TEST BUILD ONLY: the host simulation with every delta entry point, slab compaction and zone deltas.  This
// file is the translation unit of libgarecon_hostsim.so: it includes compact.cpp (hostsim.cpp + the object and AWS deltas + the
// compaction) whole and adds gar_snapshot_apply_zones, so that the CPU tier runs the zone-set splice (ActualSplicer, csrc/
// gar_delta.h) against the oracle.  Like gar_snapshot_apply_actual, it runs on the engine's ActualHost backend and DeltaHost
// buffers.
#include "compact.cpp"

extern "C" {

int gar_snapshot_apply_zones(gar_engine *e, const gar_zone_delta *d, gar_zone_delta_result *out) {
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
