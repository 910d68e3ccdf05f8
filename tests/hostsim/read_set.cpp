// read_set.cpp — TEST BUILD ONLY: the host simulation with every delta entry point, slab compaction, zone deltas, the export and
// the read set.  This file is the translation unit of libgarecon_hostsim.so: it includes export.cpp whole and adds gar_read_set,
// so that the CPU tier runs the read-set driver (ReadSetter, csrc/gar_pipeline.h) against the Python statement of the rules in
// tests/readset_ref.py.
#include <map>

#include "export.cpp"

// the read-set backend: kernels run on the engine itself; its scratch is plain host memory
struct ReadSetHost {
  gar_engine &e;
  HBuf buf[8];
  ReadSetClean clean;
  std::vector<u32> rows;
  std::vector<gar_str> strs;
  template <class F>
  void for_each(const char *name, u32 n, const F &f) { e.for_each(name, n, f); }
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
  void *read_set_buf(int k, size_t bytes) { return buf[k].ensure(bytes); }
};
static std::map<gar_engine *, ReadSetHost *> g_read_set;

extern "C" {

int gar_read_set(gar_engine *e, const gar_keyset *ks, gar_readset *out) {
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
  const int rc = R.run(e->key_rows.data(), ks->n_rows, DelKeys{e->del_kind.data(), e->del_key.data(), e->del_slab.data()}, ks->n_deleted);
  if (g_nonuniform_vote || g_vote_outside_warp) {
    e->err = "non-uniform warp vote";
    return GAR_E_STATE;
  }
  if (rc != GAR_OK) {
    e->err = "objects layout rule violated";
    return rc;
  }
  const u32 nl = R.n[RS_LB], na = R.n[RS_ACC], nz = R.n[RS_ZONE], nm = R.n[RS_MISS];
  h->rows.assign(R.out.rows[RS_LB], R.out.rows[RS_LB] + nl);
  h->rows.insert(h->rows.end(), R.out.rows[RS_ACC], R.out.rows[RS_ACC] + na);
  h->rows.insert(h->rows.end(), R.out.rows[RS_ZONE], R.out.rows[RS_ZONE] + nz);
  h->rows.insert(h->rows.end(), R.out.miss_obj, R.out.miss_obj + nm);
  h->rows.insert(h->rows.end(), R.out.miss_j, R.out.miss_j + nm);
  h->rows.push_back(0);
  h->strs.assign(R.out.miss_name, R.out.miss_name + nm);
  h->strs.insert(h->strs.end(), R.out.miss_region, R.out.miss_region + nm);
  h->strs.push_back(0);
  const u32 *r = h->rows.data();
  out->n_lbs = nl;
  out->lb_rows = r;
  out->n_accels = na;
  out->acc_rows = r + nl;
  out->n_zones = nz;
  out->zone_rows = r + nl + na;
  out->n_lb_misses = nm;
  out->lb_miss_obj = r + nl + na + nz;
  out->lb_miss_j = r + nl + na + nz + nm;
  out->lb_miss_name = h->strs.data();
  out->lb_miss_region = h->strs.data() + nm;
  return GAR_OK;
}

void gar_read_set_free(gar_engine *, gar_readset *rs) {
  if (rs) memset(rs, 0, sizeof(*rs));
}

}  // extern "C"
