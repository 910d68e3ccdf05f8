// backend_harness.cu — TEST BUILD ONLY: the CUDA backend's own primitives (csrc/gar_engine.cu) called one at a time.
//
// The host simulation (tests/hostsim) swaps every backend primitive for a serial loop, so the device-wide scan, the radix
// sort, the fused / device-counted launches and the TMA-staged string windows are otherwise only exercised through whole
// diffs.  This library compiles the engine a second time and exposes each primitive on plain host arrays: upload, call the
// engine's member function on its stream, download.  tests/test_backend_kernels.py compares the results with numpy.
// Built by __graft_entry__.build_backend_harness(); never loaded by the package.
#include "../../aws-global-accelerator-controller_b200/csrc/gar_engine.cu"

namespace {

// device buffers of one call, freed when it returns (the engine's stream is synchronised by every download)
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

// counts its visits; an index outside its own range goes to *stray instead
struct FHit {
  u32 *hits;
  u32 n;
  u32 *stray;
  __device__ void operator()(u32 i) const {
    if (i < n) atomicAdd(hits + i, 1u);
    else atomicAdd(stray, 1u);
  }
};
// the warp-synchronous form: also records `valid` and whether the whole warp was converged at the call
struct FWarpHit {
  u32 *hits;
  u8 *valid;
  u32 n;
  u32 *stray, *partial;
  __device__ void operator()(u32 i, bool v) const {
    if (__activemask() != 0xFFFFFFFFu) atomicAdd(partial, 1u);
    if (i < n) {
      atomicAdd(hits + i, 1u);
      valid[i] = v ? 1 : 0;
    } else {
      atomicAdd(stray, 1u);
    }
  }
};

// A staged row pass over caller-built string columns.  Window c of a block spans from the first row's string to the end of
// the last row's (as FTokenise / FPrepareRecord do), unless no_window[block][c] says there is none.  Every row copies the
// bytes it sees through the view for each column and records whether they came from shared memory.
template <int COLS, u32 BYTES>
struct FStageProbe {
  static constexpr int kStageCols = COLS;
  static constexpr u32 kStageBytes = BYTES;
  static constexpr bool kStageByDefault = true;
  const gar_str *refs;  // [n][2]
  const u8 *slab0, *slab1;
  const u8 *no_window;  // [blocks][2]
  const u64 *out_begin; // [n][2]: where the row's bytes of column c go in `out`
  u8 *out;
  u8 *from_smem;        // [n][2]: 1 shared memory, 0 slab
  GAR_HD const u8 *stage_slab(int c) const { return c ? slab1 : slab0; }
  GAR_HD bool stage_window(int c, u32 r0, u32 r1, u64 *lo, u64 *hi) const {
    if (no_window[(r0 / 256) * 2 + c]) return false;
    const gar_str a = refs[2 * (size_t)r0 + c], b = refs[2 * (size_t)(r1 - 1) + c];
    *lo = GAR_STR_OFF(a);
    *hi = GAR_STR_OFF(b) + GAR_STR_LEN(b);
    return true;
  }
  template <class View>
  __device__ void run(u32 i, const View &view) const {
    for (int c = 0; c < COLS; c++) {
      const Str s = view(c, refs[2 * (size_t)i + c]);
      u8 *o = out + out_begin[2 * (size_t)i + c];
      for (u32 k = 0; k < s.n; k++) o[k] = s.p[k];
      from_smem[2 * (size_t)i + c] = __isShared(s.p) ? 1 : 0;
    }
  }
  struct Direct {
    const u8 *s0, *s1;
    __device__ Str operator()(int c, gar_str r) const { return mkstr(c ? s1 : s0, r); }
  };
  __device__ void operator()(u32 i) const { run(i, Direct{slab0, slab1}); }  // the direct form (GAR_NO_TMA=1)
};

template <size_t... I>
void multi(gar_engine *e, const u32 *ns, const FHit *fs, std::index_sequence<I...>) {
  e->for_each_multi("harness_multi", {ns[I]...}, fs[I]...);
}

template <int COLS, u32 BYTES>
void staged(gar_engine *e, const gar_str *refs, u32 n, const u8 *slab0, u64 len0, u32 shift0, const u8 *slab1, u64 len1, u32 shift1,
            const u8 *no_window, const u64 *out_begin, u64 out_len, u8 *out, u8 *from_smem) {
  Scratch s;
  const u32 blocks = (n + 255) / 256;
  FStageProbe<COLS, BYTES> f{};
  gar_str *d_refs = s.alloc<gar_str>(2 * (size_t)n);
  u8 *d_s0 = s.alloc<u8>(len0 + shift0, GAR_SLAB_PAD), *d_s1 = s.alloc<u8>(len1 + shift1, GAR_SLAB_PAD);
  u8 *d_nw = s.alloc<u8>(2 * (size_t)blocks);
  u64 *d_ob = s.alloc<u64>(2 * (size_t)n);
  u8 *d_out = s.alloc<u8>(out_len), *d_fs = s.alloc<u8>(2 * (size_t)n);
  up(e, d_refs, refs, 16 * (size_t)n);
  CK(cudaMemsetAsync(d_s0, 0, len0 + shift0 + GAR_SLAB_PAD, e->stream));
  CK(cudaMemsetAsync(d_s1, 0, len1 + shift1 + GAR_SLAB_PAD, e->stream));
  up(e, d_s0 + shift0, slab0, len0);
  up(e, d_s1 + shift1, slab1, len1);
  up(e, d_nw, no_window, 2 * (size_t)blocks);
  up(e, d_ob, out_begin, 16 * (size_t)n);
  CK(cudaMemsetAsync(d_out, 0, out_len + 1, e->stream));
  CK(cudaMemsetAsync(d_fs, 0xFF, 2 * (size_t)n, e->stream));
  f.refs = d_refs;
  f.slab0 = d_s0 + shift0;
  f.slab1 = d_s1 + shift1;
  f.no_window = d_nw;
  f.out_begin = d_ob;
  f.out = d_out;
  f.from_smem = d_fs;
  e->for_each_staged("harness_staged", n, f);
  down(e, out, d_out, out_len);
  down(e, from_smem, d_fs, 2 * (size_t)n);
}

gar_engine *to_engine(void *h) { return (gar_engine *)h; }

}  // namespace

extern "C" {

int bh_create(int device, void **out) {
  gar_config cfg{GAR_ABI_VERSION, device, "harness", 0};
  gar_engine *e = nullptr;
  const int rc = gar_engine_create(&cfg, &e);
  *out = e;
  return rc;
}
void bh_destroy(void *h) { gar_engine_destroy(to_engine(h)); }
const char *bh_error(void *h) { return gar_last_error(to_engine(h)); }

// data[0..n) <- its exclusive prefix sums (mod 2^32)
int bh_exclusive_scan(void *h, u32 *data, u32 n) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    Scratch s;
    u32 *d = s.alloc<u32>(n);
    up(e, d, data, 4 * (size_t)n);
    e->exclusive_scan(d, n);
    down(e, data, d, 4 * (size_t)n);
  });
}

// stable sort of (keys, vals) by the keys' low `bits` bits as the engine passes them (result in place)
int bh_sort_pairs(void *h, u32 *keys, u32 *vals, u32 n, int bits) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    Scratch s;
    u32 *k = s.alloc<u32>(n), *v = s.alloc<u32>(n), *k2 = s.alloc<u32>(n), *v2 = s.alloc<u32>(n);
    up(e, k, keys, 4 * (size_t)n);
    up(e, v, vals, 4 * (size_t)n);
    e->sort_pairs(k, v, k2, v2, n, bits);
    down(e, keys, k, 4 * (size_t)n);
    down(e, vals, v, 4 * (size_t)n);
  });
}

// count functors (1..MULTI_MAX) over segments ns[k] in one fused launch: hits = the segments' visit counts back to back
int bh_for_each_multi(void *h, const u32 *ns, int count, u32 *hits, u32 *stray) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    if (count < 1 || count > MULTI_MAX) throw InvalidError{"count out of range"};
    Scratch s;
    size_t total = 0;
    for (int k = 0; k < count; k++) total += ns[k];
    u32 *d = s.alloc<u32>(total + 1);
    CK(cudaMemsetAsync(d, 0, 4 * (total + 2), e->stream));
    FHit fs[MULTI_MAX];
    size_t off = 0;
    for (int k = 0; k < count; k++) {
      fs[k] = FHit{d + off, ns[k], d + total};
      off += ns[k];
    }
    switch (count) {
      case 1: multi(e, ns, fs, std::make_index_sequence<1>{}); break;
      case 2: multi(e, ns, fs, std::make_index_sequence<2>{}); break;
      case 3: multi(e, ns, fs, std::make_index_sequence<3>{}); break;
      case 4: multi(e, ns, fs, std::make_index_sequence<4>{}); break;
      case 5: multi(e, ns, fs, std::make_index_sequence<5>{}); break;
      case 6: multi(e, ns, fs, std::make_index_sequence<6>{}); break;
      case 7: multi(e, ns, fs, std::make_index_sequence<7>{}); break;
      default: multi(e, ns, fs, std::make_index_sequence<8>{}); break;
    }
    down(e, hits, d, 4 * total);
    down(e, stray, d + total, 4);
  });
}

// for_each_dyn (warp = 0) or for_each_warp_dyn (warp = 1) with the count n on the device and capacity cap.  hits / valid have
// room for every thread the launch has (cap rounded up to 256).
int bh_for_each_dyn(void *h, int warp, u32 n, u32 cap, u32 *hits, u8 *valid, u32 *stray, u32 *partial) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    Scratch s;
    const size_t len = ((size_t)cap + 255) / 256 * 256;
    u32 *d = s.alloc<u32>(len + 3);
    u8 *dv = s.alloc<u8>(len);
    CK(cudaMemsetAsync(d, 0, 4 * (len + 3), e->stream));
    CK(cudaMemsetAsync(dv, 0xFF, len + 1, e->stream));
    up(e, d + len + 2, &n, 4);
    if (warp) e->for_each_warp_dyn("harness_warp_dyn", d + len + 2, cap, FWarpHit{d, dv, (u32)len, d + len, d + len + 1});
    else e->for_each_dyn("harness_dyn", d + len + 2, cap, FHit{d, (u32)len, d + len});
    down(e, hits, d, 4 * len);
    down(e, valid, dv, len);
    down(e, stray, d + len, 4);
    down(e, partial, d + len + 1, 4);
  });
}

// out[0..n + tail) starts as `sentinel`; fill32(out, v, n)
int bh_fill32(void *h, u32 v, u64 n, u32 tail, u32 sentinel, u32 *out) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    Scratch s;
    u32 *d = s.alloc<u32>(n + tail);
    e->fill32(d, sentinel, n + tail);
    e->fill32(d, v, n);
    down(e, out, d, 4 * (n + tail));
  });
}

// k_for_each_staged with an FStageProbe.  variant 0: two windows of 1 KB; 1: one window of 24 KB (the tokeniser's shape);
// 2: two windows of 16 KB (prepare_records' shape).  refs[2 * i + c] is row i's string of column c, relative to slab c, which
// sits `shift_c` bytes past a 256-byte aligned allocation.
int bh_for_each_staged(void *h, int variant, const gar_str *refs, u32 n, const u8 *slab0, u64 len0, u32 shift0, const u8 *slab1, u64 len1,
                       u32 shift1, const u8 *no_window, const u64 *out_begin, u64 out_len, u8 *out, u8 *from_smem) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    if (variant == 0) staged<2, 1024>(e, refs, n, slab0, len0, shift0, slab1, len1, shift1, no_window, out_begin, out_len, out, from_smem);
    else if (variant == 1) staged<1, 24 * 1024>(e, refs, n, slab0, len0, shift0, slab1, len1, shift1, no_window, out_begin, out_len, out, from_smem);
    else staged<2, 16 * 1024>(e, refs, n, slab0, len0, shift0, slab1, len1, shift1, no_window, out_begin, out_len, out, from_smem);
  });
}

}  // extern "C"
