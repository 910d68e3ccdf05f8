"""Host-to-device rate of gar_snapshot_load for the same tables in three placements: pageable, copied into cudaHostAlloc
memory, and generator buffers pinned in place with cudaHostRegister (what bench.py's end-to-end arm does)."""
import ctypes as C
import importlib
import sys
import time
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
import torch  # noqa: E402
import bench  # noqa: E402

pkg = importlib.import_module("aws-global-accelerator-controller_b200")
synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
abi = pkg.abi
snap = synth.generate(3, 1_000_000)
o, a = snap.objects, snap.actual


class S:
    pass


def run(label, so, sa):
    s = S()
    s.objects, s.actual = so, sa
    with pkg.Engine(cluster_name="default") as e:
        for _ in range(2):
            e.load(s)
            e.diff_raw()
        t = []
        for _ in range(5):
            t0 = time.perf_counter()
            e.load(s)
            t1 = time.perf_counter()
            r = e.diff_raw()
            t.append((r["ms_h2d"], (t1 - t0) * 1e3))
    nb = sum(int(c) * sz for (_, c, sz) in bench._table_arrays(abi, so, sa))
    h = sorted(x[0] for x in t)[2]
    w = sorted(x[1] for x in t)[2]
    print(f"{label}: H2D {h:.2f} ms = {nb / h / 1e6:.1f} GB/s, gar_snapshot_load wall {w:.2f} ms, bytes {nb / 1e6:.0f} MB")


def hostalloc_copy(so, sa):
    import copy
    o2, a2 = type(so)(), type(sa)()
    C.memmove(C.byref(o2), C.byref(so), C.sizeof(so))
    C.memmove(C.byref(a2), C.byref(sa), C.sizeof(sa))
    keep = []
    names_o = [f[0] for f in so._fields_ if not f[0].startswith("n_") and f[0] != "slab_len"]
    names_a = [f[0] for f in sa._fields_ if not f[0].startswith("n_") and f[0] != "slab_len"]
    arrays = bench._table_arrays(abi, so, sa)
    k = 0
    for st, names in ((o2, names_o), (a2, names_a)):
        for nm in names:
            ptr, cnt, sz = arrays[k]
            k += 1
            nbytes = int(cnt) * sz
            t = torch.empty(max(nbytes, 64) + 64, dtype=torch.uint8).pin_memory()
            addr = C.cast(ptr, C.c_void_p).value
            if addr and nbytes:
                C.memmove(t.data_ptr(), addr, nbytes)
            keep.append(t)
            setattr(st, nm, C.cast(t.data_ptr(), type(getattr(st, nm))))
    return o2, a2, keep


run("pageable (no pinning)", o, a)
o2, a2, keep = hostalloc_copy(o, a)
run("cudaHostAlloc copies", o2, a2)
bench._pin_host_tables(torch, abi, o, a)
run("cudaHostRegister in place", o, a)
