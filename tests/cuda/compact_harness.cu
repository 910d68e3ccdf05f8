// compact_harness.cu — TEST BUILD ONLY: the CUDA primitives of the slab compaction (csrc/gar_engine.cu) called one at a time.
//
// The host simulation runs a serial loop in place of the 64-bit look-back scan and copies a window string by string, so whole
// compactions only reach the kernels at the shapes a model happens to produce.  This library compiles the engine once more and
// exposes the two primitives on plain host arrays: upload, call the engine's member function on its stream, download.
// tests/test_compact_kernels.py compares the results with numpy.
// Built by __graft_entry__.build_backend_harness(name="compact_harness"); never loaded by the package.
#include "../../aws-global-accelerator-controller_b200/csrc/gar_engine.cu"

namespace {

// device buffers of one call, freed when it returns (the engine's stream is synchronised by every download)
struct Scratch {
  std::vector<void *> ps;
  ~Scratch() {
    for (void *p : ps) cudaFree(p);
  }
  template <class T>
  T *alloc(size_t count) {
    void *p = nullptr;
    CK(cudaMalloc(&p, count * sizeof(T) + 64));
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

int ch_create(int device, void **out) {
  gar_config cfg{GAR_ABI_VERSION, device, "harness", 0};
  gar_engine *e = nullptr;
  const int rc = gar_engine_create(&cfg, &e);
  *out = e;
  return rc;
}
void ch_destroy(void *h) { gar_engine_destroy(to_engine(h)); }
const char *ch_error(void *h) { return gar_last_error(to_engine(h)); }
uint32_t ch_window(void) { return COMPACT_WINDOW; }
uint32_t ch_long(void) { return COMPACT_LONG; }

// data[0..n) <- its exclusive prefix sums as u64
int ch_exclusive_scan64(void *h, u64 *data, u32 n) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    Scratch s;
    u64 *d = s.alloc<u64>(n);
    up(e, d, data, 8 * (size_t)n);
    e->exclusive_scan(d, n);
    down(e, data, d, 8 * (size_t)n);
  });
}

// compact_copy of m strings: sref[p] names string p inside `slab` (slab_len bytes, followed by GAR_SLAB_PAD zero bytes on the
// device), off[0..m] are the destination offsets, off[m] = total.  out has total + guard bytes and starts as 0xCD: bytes behind
// `total` must come back untouched.
int ch_compact_copy(void *h, const gar_str *sref, const u64 *off, u32 m, const u8 *slab, u64 slab_len, int any_long, u8 *out, u32 guard) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    Scratch s;
    const u64 total = off[m];
    gar_str *dref = s.alloc<gar_str>((size_t)m + 1);
    u64 *doff = s.alloc<u64>((size_t)m + 1);
    u8 *dslab = s.alloc<u8>(slab_len + GAR_SLAB_PAD), *dout = s.alloc<u8>(total + guard);
    up(e, dref, sref, 8 * (size_t)m);
    up(e, doff, off, 8 * ((size_t)m + 1));
    up(e, dslab, slab, slab_len);
    CK(cudaMemsetAsync(dslab + slab_len, 0, GAR_SLAB_PAD, e->stream));
    CK(cudaMemsetAsync(dout, 0xCD, total + guard, e->stream));
    e->compact_copy(dout, dslab, dref, doff, m, total, any_long != 0);
    down(e, out, dout, total + guard);
  });
}

}  // extern "C"
