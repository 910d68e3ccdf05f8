// export_harness.cu — TEST BUILD ONLY: the window-range copy and the pipelined gather-to-host of gar_snapshot_export
// (csrc/gar_engine.cu) called on plain host arrays, next to the compaction primitives of compact_harness.cu (included whole).
// tests/test_export_kernels.py compares the results with numpy.
// Built by __graft_entry__.build_backend_harness(name="export_harness"); never loaded by the package.
#include "compact_harness.cu"

extern "C" {

uint32_t ch_export_chunk(void) { return EXPORT_CHUNK; }
uint32_t ch_export_ring(void) { return EXPORT_RING; }

// compact_copy of windows [w0, w1) only: out receives destination bytes w0 * COMPACT_WINDOW .. min(w1 * COMPACT_WINDOW, total)
// followed by `guard` bytes that start as 0xCD and must come back untouched
int ch_compact_copy_range(void *h, const gar_str *sref, const u64 *off, u32 m, const u8 *slab, u64 slab_len, int any_long, u32 w0, u32 w1,
                          u8 *out, u64 out_len, u32 guard) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    Scratch s;
    gar_str *dref = s.alloc<gar_str>((size_t)m + 1);
    u64 *doff = s.alloc<u64>((size_t)m + 1);
    u8 *dslab = s.alloc<u8>(slab_len + GAR_SLAB_PAD), *dout = s.alloc<u8>(out_len + guard);
    up(e, dref, sref, 8 * (size_t)m);
    up(e, doff, off, 8 * ((size_t)m + 1));
    up(e, dslab, slab, slab_len);
    CK(cudaMemsetAsync(dslab + slab_len, 0, GAR_SLAB_PAD, e->stream));
    CK(cudaMemsetAsync(dout, 0xCD, out_len + guard, e->stream));
    e->compact_copy(dout, dslab, dref, doff, m, off[m], any_long != 0, w0, w1);
    down(e, out, dout, out_len + guard);
  });
}

// the export's gather of the whole slab, chunk by chunk through the ring, into the host array out (total + guard bytes,
// pageable or pinned by the caller); guard bytes must come back untouched
int ch_export_slab(void *h, const gar_str *sref, const u64 *off, u32 m, const u8 *slab, u64 slab_len, int any_long, u8 *out) {
  gar_engine *e = to_engine(h);
  return guarded(e, [&] {
    Scratch s;
    gar_str *dref = s.alloc<gar_str>((size_t)m + 1);
    u64 *doff = s.alloc<u64>((size_t)m + 1);
    u8 *dslab = s.alloc<u8>(slab_len + GAR_SLAB_PAD);
    up(e, dref, sref, 8 * (size_t)m);
    up(e, doff, off, 8 * ((size_t)m + 1));
    up(e, dslab, slab, slab_len);
    CK(cudaMemsetAsync(dslab + slab_len, 0, GAR_SLAB_PAD, e->stream));
    e->export_fence();
    const int rc = e->export_slab(out, dslab, dref, doff, m, off[m], any_long != 0);
    e->export_end();
    if (rc != GAR_OK) throw DeviceMemoryError{"no ring"};
  });
}

}  // extern "C"
