// shard_pack_harness.cu — TEST BUILD ONLY: the sharded exchange's data-path kernels (csrc/gar_shard.h, gar_engine.cu) called
// one at a time on caller-built inputs.
//
// Whole exchanges of small models never reach the shapes where these kernels branch (a block straddling two destinations, a
// block range of exactly PACK_TILE bytes, strings cut at SH_LONG_WORDS, the second stride of FShPackLong, the remainder loop of
// k_peer_push).  This library compiles the engine a second time and exposes
//   sph_pack   one level of one source rank packed into G destinations: the level plan is built the way route + plan_finish
//              build it (FShRowSizes, the engine's exclusive scans, FShDerivedBounds), then Sharder::pack_to runs the level
//              with the default pack (k_for_each<FShPackRows> + FShPackLong) or the bulk-store pack (k_shard_pack_rows +
//              FShPackLong), into a caller buffer that starts as a sentinel byte
//   sph_push   k_peer_push on 1..GAR_SHARD_MAX_RANKS descriptors, each destination sentinel-filled with guard bands around it
// tests/test_shard_pack_kernels.py compares every byte with a numpy restatement of the blob layout (tests/shardblob.py).
// Built by __graft_entry__.build_backend_harness(name="shard_pack_harness"); never loaded by the package.
#include "../../aws-global-accelerator-controller_b200/csrc/gar_engine.cu"

namespace {

struct Scratch {
  std::vector<void *> ps;
  ~Scratch() {
    for (void *p : ps) cudaFree(p);
  }
  template <class T>
  T *alloc(size_t count, size_t extra_bytes = 0) {
    void *p = nullptr;
    CK(cudaMalloc(&p, count * sizeof(T) + extra_bytes + 16));
    ps.push_back(p);
    return (T *)p;
  }
};
void up(gar_engine *e, void *dst, const void *src, size_t bytes) {
  if (bytes) CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, e->stream));
}
void down(gar_engine *e, void *dst, const void *src, size_t bytes) {
  if (bytes) CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaGetLastError());
}

gar_engine *to_engine(void *h) { return (gar_engine *)h; }

}  // namespace

extern "C" {

int sph_create(int device, void **out) {
  gar_config cfg{GAR_ABI_VERSION, device, "harness", 0};
  gar_engine *e = nullptr;
  const int rc = gar_engine_create(&cfg, &e);
  *out = e;
  return rc;
}
void sph_destroy(void *h) { gar_engine_destroy(to_engine(h)); }
const char *sph_error(void *h) { return gar_last_error(to_engine(h)); }

// Constants the Python side restates; returned so a change here fails the test instead of silently shifting its shapes.
void sph_constants(u64 *out) {
  out[0] = PACK_TILE;
  out[1] = SH_LONG_WORDS;
  out[2] = SH_LONG_WORKERS;
  out[3] = SH_COPY_LANES;
  out[4] = (u64)PUSH_BLOCKS * PUSH_THREADS;
  out[5] = GAR_SLAB_PAD;
  out[6] = L_NLEVELS;
}

// Pack level `lvl` of n source rows.  Source columns (host arrays, the level's schema decides which are read):
//   str [n_str][n] string refs into slab (slab_len bytes, uploaded to a 256-byte aligned buffer followed by GAR_SLAB_PAD bytes
//   of `pad_byte`), u8c [n_u8][n], u32c [n_u32][n], gid [n] or null (then gid_base + row), child_begin [n_child][n + 1].
// Selection: sel[m] grouped by destination, row_off[G + 1].  Destination d's level starts at byte dst_off[d] (16-aligned) of
// `out` (out_len bytes, all `sentinel` before the pack).  tma = 1 packs with k_shard_pack_rows.  Returns the plan's slab_scan
// (m + 1 entries) in scan_out.
int sph_pack(void *h, int lvl, int tma, u32 G, const u8 *slab, u64 slab_len, u8 pad_byte, const u64 *str, const u8 *u8c, const u32 *u32c,
             const u32 *gid, u32 gid_base, const u32 *child_begin, u32 n, const u32 *sel, u32 m, const u32 *row_off, const u64 *dst_off,
             u8 sentinel, u64 out_len, u8 *out, u32 *scan_out) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    if (lvl < 0 || lvl >= L_NLEVELS || G < 1 || G > SH_MAX_RANKS) throw InvalidError{"bad level or destination count"};
    for (u32 d = 0; d < G; d++)
      if (dst_off[d] & 15) throw InvalidError{"destination offsets must be 16-byte aligned"};
    const LevelSchema &S = SH_SCHEMA[lvl];
    Scratch s;
    u8 *d_slab = s.alloc<u8>(slab_len, GAR_SLAB_PAD);
    up(e, d_slab, slab, slab_len);
    CK(cudaMemsetAsync(d_slab + slab_len, pad_byte, GAR_SLAB_PAD, e->stream));
    LevelSrc src{};
    src.slab = d_slab;
    src.n = n;
    src.gid_base = gid_base;
    for (int c = 0; c < S.n_str; c++) {
      gar_str *p = s.alloc<gar_str>(n);
      up(e, p, str + (size_t)c * n, 8 * (size_t)n);
      src.str[c] = p;
    }
    for (int c = 0; c < S.n_u8; c++) {
      u8 *p = s.alloc<u8>(n);
      up(e, p, u8c + (size_t)c * n, n);
      src.u8c[c] = p;
    }
    for (int c = 0; c < S.n_u32; c++) {
      u32 *p = s.alloc<u32>(n);
      up(e, p, u32c + (size_t)c * n, 4 * (size_t)n);
      src.u32c[c] = p;
    }
    if (S.has_gid && gid) {
      u32 *p = s.alloc<u32>(n);
      up(e, p, gid, 4 * (size_t)n);
      src.gid = p;
    }
    for (int c = 0; c < S.n_child; c++) {
      u32 *p = s.alloc<u32>((size_t)n + 1);
      up(e, p, child_begin + (size_t)c * (n + 1), 4 * ((size_t)n + 1));
      src.child_begin[c] = p;
    }
    u8 *d_out = s.alloc<u8>(out_len);
    CK(cudaMemsetAsync(d_out, sentinel, out_len, e->stream));

    // the plan of one level, as Sharder::set_top + plan_children_and_strings leave it (the child levels' own plans are not built)
    Sharder<gar_engine> sh(*e);
    sh.G = G;
    sh.plan_begin();
    sh.active[lvl] = true;
    sh.src[lvl] = src;
    LevelPlan &P = sh.plan[lvl];
    P.cap = m;
    P.m = sh.m_dev(lvl);
    P.row_off = sh.row_off_dev(lvl);
    P.slab_off = sh.slab_off_dev(lvl);
    P.sel = sh.alloc<u32>(SH_ARENA_PLAN, m);
    up(e, P.sel, sel, 4 * (size_t)m);
    up(e, P.row_off, row_off, 4 * ((size_t)G + 1));
    up(e, P.m, &m, 4);
    for (int c = 0; c < S.n_child; c++) P.cnt[c] = sh.alloc<u32>(SH_ARENA_PLAN, (size_t)m + 1);
    P.slab_scan = sh.alloc<u32>(SH_ARENA_PLAN, (size_t)m + 1);
    e->for_each("shard_row_sizes", m + 1, FShRowSizes{src, S, P, G});
    for (int c = 0; c < S.n_child; c++) e->exclusive_scan(P.cnt[c], m + 1);
    if (S.n_str) e->exclusive_scan(P.slab_scan, m + 1);
    e->for_each("shard_slab_bounds", G + 1, FShDerivedBounds{P.row_off, P.slab_scan, G, P.slab_off, nullptr});
    std::vector<u32> hb(2 * (SH_MAX_RANKS + 1));
    down(e, hb.data(), P.row_off, 4 * hb.size());
    for (u32 d = 0; d <= G; d++) {
      sh.h_row_off[lvl][d] = hb[d];
      sh.h_slab_off[lvl][d] = hb[SH_MAX_RANKS + 1 + d];
    }
    // pack_to lays the levels out from offset 0 of every destination: with the levels before `lvl` empty, `lvl` starts at the base
    u8 *bases[SH_MAX_RANKS] = {};
    for (u32 d = 0; d < G; d++) bases[d] = d_out + dst_off[d];
    const bool tma0 = e->pack_tma;
    e->pack_tma = tma != 0;
    try {
      sh.pack_to(bases);
    } catch (...) {
      e->pack_tma = tma0;
      throw;
    }
    e->pack_tma = tma0;
    down(e, out, d_out, out_len);
    down(e, scan_out, P.slab_scan, 4 * ((size_t)m + 1));
  });
}

// k_peer_push over `cnt` descriptors: descriptor k copies n16[k] uint4 from src (host, back to back) into a destination that
// sits `guard` bytes (a multiple of 16) into a buffer of guard + 16 n16[k] + guard bytes, all `sentinel` before the launch.
// out receives every destination buffer, guards included, back to back.
int sph_push(void *h, int cnt, const u64 *n16, const u8 *src, u64 guard, u8 sentinel, u8 *out) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    if (cnt < 1 || cnt > GAR_SHARD_MAX_RANKS || (guard & 15)) throw InvalidError{"bad descriptor count or guard"};
    Scratch s;
    PushDesc pd{};
    u8 *dsts[GAR_SHARD_MAX_RANKS] = {};
    u64 src_off = 0;
    for (int k = 0; k < cnt; k++) {
      const u64 bytes = 16 * n16[k];
      u8 *ds = s.alloc<u8>(bytes), *dd = s.alloc<u8>(bytes + 2 * guard);
      up(e, ds, src + src_off, bytes);
      CK(cudaMemsetAsync(dd, sentinel, bytes + 2 * guard, e->stream));
      pd.src[k] = (const uint4 *)ds;
      pd.dst[k] = (uint4 *)(dd + guard);
      pd.n16[k] = n16[k];
      dsts[k] = dd;
      src_off += bytes;
    }
    k_peer_push<<<dim3(PUSH_BLOCKS, cnt), PUSH_THREADS, 0, e->stream>>>(pd);
    CK(cudaGetLastError());
    u64 out_off = 0;
    for (int k = 0; k < cnt; k++) {
      const u64 bytes = 16 * n16[k] + 2 * guard;
      down(e, out + out_off, dsts[k], bytes);
      out_off += bytes;
    }
  });
}

}  // extern "C"
