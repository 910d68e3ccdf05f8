// record_deltas.cpp — TEST BUILD ONLY: the host simulation with every delta entry point, slab compaction, zone deltas, the export,
// the read set and the record deltas.  This file is the translation unit of libgarecon_hostsim.so: it includes read_set.cpp whole
// and adds gar_snapshot_apply_records (the record splice of ActualSplicer, csrc/gar_delta.h, on the engine's ActualHost backend
// and DeltaHost buffers, as gar_snapshot_apply_zones runs) and gar_read_records (ReadSetter's record mode, csrc/gar_pipeline.h,
// on the ReadSetHost backend of gar_read_set).
#include "read_set.cpp"

static std::map<gar_engine *, std::vector<u32> *> g_read_records;

extern "C" {

int gar_snapshot_apply_records(gar_engine *e, const gar_record_delta *d, gar_record_delta_result *out) {
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

int gar_read_records(gar_engine *e, const gar_keyset *ks, gar_record_readset *out) {
  if (!e || !ks || !out) return GAR_E_INVALID;
  memset(out, 0, sizeof(*out));
  if (!e->loaded || e->shard_home || e->shard_round != 0) {
    e->err = "no snapshot loaded, or sharded mode";
    return GAR_E_STATE;
  }
  if ((ks->n_rows && !ks->rows) || (ks->n_deleted && (!ks->deleted_kind || !ks->deleted_key))) {
    e->err = "NULL key set arrays";
    return GAR_E_INVALID;
  }
  for (u32 k = 0; k < ks->n_rows; k++)
    if (ks->rows[k] >= e->T.o.n_objects) {
      e->err = "key set row out of range";
      return GAR_E_INVALID;
    }
  for (u32 k = 0; k < ks->n_deleted; k++)
    if (!ks->deleted_key[k] || ks->deleted_kind[k] > GAR_KIND_INGRESS) {
      e->err = "bad deleted key";
      return GAR_E_INVALID;
    }
  if (!e->pipe) {  // as diff_impl creates it
    e->pipe = new Pipeline<gar_engine>(*e, e->T);
    if (const char *tc = getenv("GAR_TINY_CAPS")) e->pipe->tiny_caps = tc[0] == '1';
  }
  ReadSetHost *&h = g_read_set[e];
  if (!h) h = new ReadSetHost{*e, {}, {}, {}, {}};
  std::vector<u32> *&rows = g_read_records[e];
  if (!rows) rows = new std::vector<u32>();
  // the keyed diff's staging of the key batch
  e->key_rows.assign(ks->rows, ks->rows + ks->n_rows);
  e->key_rows.push_back(0);
  e->del_slab.clear();
  e->del_key.assign(ks->n_deleted + 1, 0);
  e->del_kind.assign(ks->n_deleted + 1, 0);
  for (u32 k = 0; k < ks->n_deleted; k++) {
    size_t len = strlen(ks->deleted_key[k]);
    e->del_key[k] = GAR_STR(e->del_slab.size(), len);
    e->del_slab.insert(e->del_slab.end(), ks->deleted_key[k], ks->deleted_key[k] + len);
    e->del_kind[k] = ks->deleted_kind[k];
  }
  e->del_slab.resize(e->del_slab.size() + 64, 0);
  Pipeline<gar_engine> &P = *e->pipe;
  P.orphan_sweep = !(e->flags & GAR_FLAG_NO_ORPHANS);
  P.allow_empty_cache = (e->flags & GAR_FLAG_ALLOW_EMPTY_CACHE) != 0;
  if (e->flags & GAR_FLAG_REPREPARE) P.prepared = false;
  g_vote_outside_warp = g_nonuniform_vote = false;
  ReadSetter<ReadSetHost, Pipeline<gar_engine>> R{*h, P, h->clean};
  R.records = true;
  const int rc = R.run(e->key_rows.data(), ks->n_rows, DelKeys{e->del_kind.data(), e->del_key.data(), e->del_slab.data()}, ks->n_deleted);
  if (g_nonuniform_vote || g_vote_outside_warp) {
    e->err = "non-uniform warp vote";
    return GAR_E_STATE;
  }
  if (rc != GAR_OK) {
    e->err = "objects layout rule violated";
    return rc;
  }
  rows->assign(R.out.rows[RS_REC], R.out.rows[RS_REC] + R.n[RS_REC]);
  rows->push_back(0);
  out->n_records = R.n[RS_REC];
  out->rec_rows = rows->data();
  return GAR_OK;
}

void gar_read_records_free(gar_engine *, gar_record_readset *rs) {
  if (rs) memset(rs, 0, sizeof(*rs));
}

}  // extern "C"
