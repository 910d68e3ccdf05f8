// hostsim.cpp — TEST BUILD ONLY: the engine's row logic and pipeline (csrc/gar_rows.h, gar_pipeline.h) compiled
// for the host, with loops / std::stable_sort standing in for kernels.  It exists because the build container has
// no GPU: it lets `pytest -m "not gpu"` run the very functions the sm_90a kernels are made of against the oracle.
// It is never loaded by the package and is not a fallback: libgarecon.so has no CPU path.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

#include <condition_variable>
#include <mutex>
#include <thread>

#include "../../aws-global-accelerator-controller_b200/csrc/gar_pipeline.h"
#include "../../aws-global-accelerator-controller_b200/csrc/gar_shard.h"

// ---- warp emulation: for_each_warp runs every group of 32 lanes on 32 host threads; GAR_ANY is a barrier vote.
// A vote that not all 32 lanes reach (a lane finished, or never arrives) would hang the real GPU: here it is
// detected and reported, so vote-uniformity of the device code is checked on the CPU tier.
struct WarpCtx {
  std::mutex m;
  std::condition_variable cv;
  int arrived = 0, finished = 0;
  unsigned generation = 0;
  bool acc = false, result = false, error = false;
  bool vote(bool p) {
    std::unique_lock<std::mutex> lk(m);
    if (error) return false;
    if (finished > 0) {  // a lane already left the kernel: this vote can never complete on a GPU
      error = true;
      cv.notify_all();
      return false;
    }
    acc = acc || p;
    if (++arrived == 32) {
      result = acc;
      acc = false;
      arrived = 0;
      generation++;
      cv.notify_all();
      return result;
    }
    unsigned gen = generation;
    cv.wait(lk, [&] { return generation != gen || error; });
    return error ? false : result;
  }
  void finish() {
    std::unique_lock<std::mutex> lk(m);
    finished++;
    if (arrived > 0) {  // others are waiting in a vote this lane will never join
      error = true;
      cv.notify_all();
    }
  }
};
static thread_local WarpCtx *tl_warp = nullptr;
static bool g_vote_outside_warp = false, g_nonuniform_vote = false;
bool gar_host_vote(bool p) {
  if (!tl_warp) {
    g_vote_outside_warp = true;  // GAR_ANY used in a kernel that is not warp-synchronous
    return p;
  }
  return tl_warp->vote(p);
}

struct HBuf {
  std::vector<uint64_t> mem;
  void *ensure(size_t bytes) {
    size_t w = (bytes + 7) / 8 + 8;
    if (mem.size() < w) mem.assign(w, 0);
    return mem.data();
  }
};

struct gar_engine {
  std::string cluster, err;
  std::vector<uint8_t> cluster_pad;
  DevTables T{};
  bool loaded = false;
  std::vector<std::vector<uint8_t>> slabs;
  HBuf slot[S_NSLOTS];
  HBuf o_status_ga, o_status_r53, o_derived, o_ops, o_tok_code, o_tok_name, o_tok_region, o_dport_begin, o_dports, o_derived_keys;
  Pipeline<gar_engine> *pipe = nullptr;
  Sharder<gar_engine> *sharder = nullptr;
  DevTables slice{};
  bool shard_home = false;
  int shard_round = 0;
  std::vector<uint64_t> peer_arena[2];
  u8 *peer_ptr[2][GAR_SHARD_MAX_RANKS] = {};
  std::vector<HBuf> arena[3];
  size_t arena_used[3] = {0, 0, 0};
  void *shard_alloc(int a, size_t bytes) {
    if (arena_used[a] >= arena[a].size()) arena[a].emplace_back();
    return arena[a][arena_used[a]++].ensure(bytes + 32);
  }
  void shard_reset(int a) { arena_used[a] = 0; }
  void copy_bytes(void *dst, const void *src, size_t n) { memcpy(dst, src, n); }
  std::vector<u8> del_slab, del_kind;
  std::vector<gar_str> del_key;
  std::vector<u32> key_rows;
  u64 input_bytes = 0;
  u32 launches = 0;
  u32 flags = 0;

  template <class F>
  void for_each(const char *, u32 n, const F &f) {
    launches++;
    for (u32 i = 0; i < n; i++) f(i);
  }
  template <class F>
  void for_each_warp(const char *, u32 n, const F &f) {
    launches++;
    for (u32 base = 0; base < n; base += 32) {
      WarpCtx ctx;
      std::thread lanes[32];
      for (u32 l = 0; l < 32; l++)
        lanes[l] = std::thread([&, l] {
          tl_warp = &ctx;
          f(base + l, base + l < n);
          ctx.finish();
          tl_warp = nullptr;
        });
      for (auto &t : lanes) t.join();
      if (ctx.error) g_nonuniform_vote = true;
    }
  }
  template <class F>
  void for_each_staged(const char *name, u32 n, const F &f) {
    for_each(name, n, f);  // no shared memory on the host: the functor's direct form
  }
  template <class F>
  void for_each_dyn(const char *name, const u32 *n_dev, u32 cap, const F &f) {
    for_each(name, *n_dev < cap ? *n_dev : cap, f);
  }
  template <class F>
  void for_each_warp_dyn(const char *name, const u32 *n_dev, u32 cap, const F &f) {
    for_each_warp(name, *n_dev < cap ? *n_dev : cap, f);
  }
  template <class... Fs>
  void for_each_multi(const char *, std::initializer_list<u32> ns, const Fs &...fs) {
    launches++;
    auto it = ns.begin();
    auto one = [](u32 n, const auto &f) {
      for (u32 i = 0; i < n; i++) f(i);
    };
    (one(*it++, fs), ...);
  }
  int graph_begin(u64) { return 0; }
  void graph_end() {}
  void fill32(u32 *p, u32 v, size_t n) { std::fill(p, p + n, v); }
  void copy32(u32 *d, const u32 *s, size_t n) { memcpy(d, s, n * 4); }
  void exclusive_scan(u32 *d, u32 n) {
    u32 run = 0;
    for (u32 i = 0; i < n; i++) {
      u32 v = d[i];
      d[i] = run;
      run += v;
    }
  }
  // stable by the key's low 8 * ceil(bits / 8) bits: exactly what the GPU's 8-bit LSD passes see, so a caller whose keys
  // exceed its `bits` is wrong here as well
  void sort_pairs(u32 *keys, u32 *vals, u32 *, u32 *, u32 n, int bits) {
    const int seen = 8 * ((bits + 7) / 8);
    const u32 mask = seen >= 32 ? 0xFFFFFFFFu : (1u << seen) - 1u;
    std::vector<u32> idx(n);
    std::iota(idx.begin(), idx.end(), 0u);
    std::stable_sort(idx.begin(), idx.end(), [&](u32 a, u32 b) { return (keys[a] & mask) < (keys[b] & mask); });
    std::vector<u32> k(n), v(n);
    for (u32 i = 0; i < n; i++) {
      k[i] = keys[idx[i]];
      v[i] = vals[idx[i]];
    }
    memcpy(keys, k.data(), n * 4);
    memcpy(vals, v.data(), n * 4);
  }
  void *ensure(int s, size_t bytes) { return slot[s].ensure(bytes); }
  void download(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
  uint64_t dl_stage[2][4] = {};
  void download_start(int id, const void *src, size_t bytes) { memcpy(dl_stage[id], src, bytes); }
  void download_wait(int id, void *dst, size_t bytes) { memcpy(dst, dl_stage[id], bytes); }
  void *out_derived(u32 n) { return o_derived.ensure(4 * (size_t)(n + 1)); }
  void *out_derived_keys(u32 n) { return o_derived_keys.ensure(4 * (size_t)(n + 1)); }
  void *out_dport_begin(u32 n) { return o_dport_begin.ensure(4 * (size_t)(n + 2)); }
  void *out_tok_code(u32 n) { return o_tok_code.ensure(n + 1); }
  void *out_tok_name(u32 n) { return o_tok_name.ensure(8 * (size_t)(n + 1)); }
  void *out_tok_region(u32 n) { return o_tok_region.ensure(8 * (size_t)(n + 1)); }
  void *out_dports(u64 n) { return o_dports.ensure(4 * (size_t)(n + 1)); }
  void *out_status_ga(u32 n) { return o_status_ga.ensure(4 * (size_t)(n + 1)); }
  void *out_status_r53(u32 n) { return o_status_r53.ensure(4 * (size_t)(n + 1)); }
};

static std::string g_err;

extern "C" {

int gar_engine_create(const gar_config *cfg, gar_engine **out) {
  auto *e = new gar_engine();
  e->cluster = cfg->cluster_name ? cfg->cluster_name : "";
  e->flags = cfg->flags;
  e->cluster_pad.assign(e->cluster.size() + 64, 0);
  memcpy(e->cluster_pad.data(), e->cluster.data(), e->cluster.size());
  *out = e;
  return GAR_OK;
}
void gar_engine_destroy(gar_engine *e) { delete e; }

int gar_snapshot_load(gar_engine *e, const gar_objects *o, const gar_actual *a) {
  // copy only the slabs (for padding); columns are read in place (the caller keeps them alive in tests)
  e->slabs.clear();
  e->slabs.emplace_back(o->slab_len + 64, 0);
  if (o->slab_len) memcpy(e->slabs[0].data(), o->slab, o->slab_len);
  e->slabs.emplace_back(a->slab_len + 64, 0);
  if (a->slab_len) memcpy(e->slabs[1].data(), a->slab, a->slab_len);
  e->T.o = *o;
  e->T.a = *a;
  e->T.o.slab = e->slabs[0].data();
  e->T.a.slab = e->slabs[1].data();
  e->T.cluster = e->cluster_pad.data();
  e->T.cluster_len = (u32)e->cluster.size();
  e->loaded = true;
  delete e->pipe;
  e->pipe = nullptr;
  e->slice = e->T;
  e->shard_home = false;
  e->shard_round = 0;
  return GAR_OK;
}
int gar_snapshot_attach_device(gar_engine *e, const gar_objects *o, const gar_actual *a) { return gar_snapshot_load(e, o, a); }

static int diff_impl(gar_engine *e, gar_changeset *out, const gar_keyset *ks, const gar_bindings *bd = nullptr) {
  memset(out, 0, sizeof(*out));
  e->launches = 0;
  if (e->shard_home && e->shard_round != 4) return GAR_E_STATE;  // mid-exchange: the old sub-snapshot's receive buffers are being refilled
  if (!e->pipe) {
    e->pipe = new Pipeline<gar_engine>(*e, e->T);
    if (const char *tc = getenv("GAR_TINY_CAPS")) e->pipe->tiny_caps = tc[0] == '1';
    if (e->shard_home) {
      e->pipe->acc_guest_from = e->sharder->guest_from;
      e->pipe->sharded = 1;
    }
  }
  Pipeline<gar_engine> &P = *e->pipe;
  P.orphan_sweep = !(e->flags & GAR_FLAG_NO_ORPHANS);
  P.allow_empty_cache = (e->flags & GAR_FLAG_ALLOW_EMPTY_CACHE) != 0;
  DiffCounts dc{};
  g_vote_outside_warp = g_nonuniform_vote = false;
  auto ops_alloc = [&](u64 nops) { return e->o_ops.ensure(sizeof(gar_op) * (size_t)(nops + 1)); };
  int rc;
  u32 n_out = e->T.o.n_objects;
  std::vector<uint8_t> bslab;
  if (bd) {
    gar_bindings d = *bd;
    bslab.assign(bd->slab, bd->slab + bd->slab_len);
    bslab.resize(bslab.size() + 64, 0);
    d.slab = bslab.data();
    n_out = bd->n_bindings;
    rc = P.run_bindings(d, &dc, ops_alloc);
  } else if (!ks) {
    rc = P.run(&dc, ops_alloc);
  } else {
    n_out = ks->n_rows;
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
    rc = P.run_keys(e->key_rows.data(), ks->n_rows, DelKeys{e->del_kind.data(), e->del_key.data(), e->del_slab.data()}, ks->n_deleted, &dc, ops_alloc);
  }
  if (rc == GAR_OK && e->shard_home && dc.n_ops) e->for_each("shard_translate_ops", (u32)dc.n_ops, FShTranslateOps{(gar_op *)e->o_ops.mem.data(), e->sharder->gids});
  if (g_nonuniform_vote || g_vote_outside_warp) {
    e->err = g_nonuniform_vote ? "non-uniform warp vote: some lane did not reach a GAR_ANY that others executed (would hang on the GPU)"
                               : "GAR_ANY executed outside a warp-synchronous kernel";
    return GAR_E_STATE;
  }
  if (rc == GAR_REFUSE_EMPTY_CACHE) {
    e->err = "the object table is empty but this cluster still owns AWS resources: refusing to emit delete-everything orphan sections";
    return GAR_E_STATE;
  }
  if (rc != GAR_OK) {
    e->err = "objects layout rule violated";
    return rc;
  }
  out->n_objects = n_out;
  out->status_ga = (const u32 *)e->o_status_ga.mem.data();
  out->status_r53 = (const u32 *)e->o_status_r53.mem.data();
  out->derived = (const u32 *)(ks ? e->o_derived_keys.mem.data() : e->o_derived.mem.data());
  out->n_ops = dc.n_ops;
  out->ops = (const gar_op *)e->o_ops.mem.data();
  for (int k = 0; k <= GAR_N_SECTIONS; k++) out->section_begin[k] = dc.section_begin[k];
  out->n_lbi = (ks || bd) ? 0 : e->T.o.n_lbi;
  out->tok_code = (const u8 *)e->o_tok_code.mem.data();
  out->tok_name = (const gar_str *)e->o_tok_name.mem.data();
  out->tok_region = (const gar_str *)e->o_tok_region.mem.data();
  out->dport_begin = (const u32 *)e->o_dport_begin.mem.data();
  out->n_dports = dc.n_dports;
  out->dports = (const i32 *)e->o_dports.mem.data();
  out->kernel_launches = e->launches;
  out->obj_gid = e->shard_home ? e->sharder->gids.obj : nullptr;
  return GAR_OK;
}
int gar_diff(gar_engine *e, gar_changeset *out) { return diff_impl(e, out, nullptr); }
int gar_diff_keys(gar_engine *e, const gar_keyset *ks, gar_changeset *out) { return diff_impl(e, out, ks); }
int gar_bindings_diff(gar_engine *e, const gar_bindings *bd, gar_changeset *out) { return diff_impl(e, out, nullptr, bd); }
int gar_diff_device(gar_engine *e, gar_changeset *out) { return gar_diff(e, out); }
int gar_shard_route(gar_engine *e, const gar_shard *shard, int round, uint64_t *meta, uint64_t *send_bytes) {
  if (!e->sharder) e->sharder = new Sharder<gar_engine>(*e);
  if (round == 1) {
    e->sharder->route1(e->slice, *shard, meta, send_bytes);
    e->shard_round = 1;
  } else {
    if (e->shard_round != 2) return GAR_E_STATE;
    e->sharder->route2(meta, send_bytes);
    e->shard_round = 3;
  }
  return GAR_OK;
}
int gar_shard_pack(gar_engine *e, void *send) {
  e->sharder->pack((u8 *)send);
  return GAR_OK;
}
int gar_shard_unpack(gar_engine *e, int round, const void *recv, const uint64_t *recv_meta) {
  if (round == 1 && e->shard_round == 1) {
    if (e->sharder->unpack1((const u8 *)recv, recv_meta) != GAR_OK) {
      e->err = e->sharder->contract_error;
      return GAR_E_INVALID;
    }
    e->shard_round = 2;
  } else if (round == 2 && e->shard_round == 3) {
    if (e->sharder->unpack2((const u8 *)recv, recv_meta) != GAR_OK) {
      e->err = e->sharder->contract_error;
      return GAR_E_INVALID;
    }
    delete e->pipe;
    e->pipe = nullptr;
    e->T = e->sharder->H;
    e->shard_home = true;
    e->shard_round = 4;
  } else {
    return GAR_E_STATE;
  }
  return GAR_OK;
}
uint64_t gar_shard_blob_bytes(const uint64_t *meta_row) { return blob_bytes(meta_row); }
// peer-memory exchange on the host build: every "rank" lives in this process, a handle is just the arena's address
int gar_shard_arena(gar_engine *e, int round, uint64_t need_bytes, void **arena, uint8_t *handle, uint64_t *capacity) {
  std::vector<uint64_t> &b = e->peer_arena[round - 1];
  if (b.size() * 8 < need_bytes + 64) b.assign((need_bytes + need_bytes / 4 + 4096) / 8, 0);
  uint64_t p = (uint64_t)(uintptr_t)b.data();
  memset(handle, 0, GAR_SHARD_HANDLE_BYTES);
  memcpy(handle, &p, 8);
  *arena = b.data();
  if (capacity) *capacity = b.size() * 8;
  return GAR_OK;
}
int gar_shard_open_peers(gar_engine *e, int round, const uint8_t *handles) {
  for (u32 k = 0; k < e->sharder->G; k++) {
    uint64_t p;
    memcpy(&p, handles + (size_t)k * GAR_SHARD_HANDLE_BYTES, 8);
    e->peer_ptr[round - 1][k] = (u8 *)(uintptr_t)p;
  }
  return GAR_OK;
}
int gar_shard_pack_peers(gar_engine *e, int round, const uint64_t *all_meta) {
  const u32 G = e->sharder->G, me = e->sharder->cfg.rank;
  u8 *bases[GAR_SHARD_MAX_RANKS] = {};
  for (u32 d = 0; d < G; d++) {
    u64 off = 0;
    for (u32 s = 0; s < me; s++) off += blob_bytes(all_meta + ((size_t)s * G + d) * GAR_SHARD_META_WORDS);
    bases[d] = e->peer_ptr[round - 1][d] + off;
  }
  e->sharder->pack_to(bases);
  return GAR_OK;
}
void gar_changeset_free(gar_engine *, gar_changeset *cs) { memset(cs, 0, sizeof(*cs)); }
const char *gar_last_error(const gar_engine *e) { return e ? e->err.c_str() : g_err.c_str(); }
const char *gar_version(void) { return "garecon hostsim (test build)"; }
uint64_t gar_algorithmic_bytes(const gar_engine *, const gar_changeset *) { return 0; }
uint32_t gar_last_stage_timings(gar_engine *, gar_stage_timing *, uint32_t) { return 0; }
uint32_t gar_last_counters(gar_engine *e, uint64_t *out, uint32_t cap) {
  if (!e || !out || cap < GAR_CTR_N) return 0;
  out[GAR_CTR_R53_PAIRS] = e->pipe ? e->pipe->n_pairs : 0;
  out[GAR_CTR_DPORTS] = e->pipe ? e->pipe->n_dports : 0;
  out[GAR_CTR_LAUNCH_MODE] = 0;  // graph_begin above never records or replays
  return GAR_CTR_N;
}
}
