"""ctypes mirror of include/garecon.h and the loader for libgarecon.so.

This is host plumbing over the C ABI (the drop-in boundary): the structs below are field-for-field the
ones in include/garecon.h.  There is no CPU fallback: if the CUDA library is missing or no sm_90 device
is present, `Engine()` raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

PKG_DIR = Path(__file__).resolve().parent
REPO = PKG_DIR.parent
LIB_PATH = PKG_DIR / "libgarecon.so"

GAR_ABI_VERSION = 1
GAR_NONE = 0xFFFFFFFF
OFF_BITS = 40
OFF_MASK = (1 << OFF_BITS) - 1

# enums (include/garecon.h)
KIND_SERVICE, KIND_INGRESS = 0, 1
SVC_CLUSTERIP, SVC_NODEPORT, SVC_LOADBALANCER, SVC_EXTERNALNAME = 0, 1, 2, 3
OBJ_HAS_LB_CLASS, OBJ_HAS_INGRESS_CLASS = 1, 2
LB_ACTIVE, LB_PROVISIONING, LB_ACTIVE_IMPAIRED, LB_FAILED = 0, 1, 2, 3
PROTO_TCP, PROTO_UDP = 0, 1
RR_OTHER, RR_A, RR_TXT, RR_CNAME, RR_AAAA = 0, 1, 2, 3, 4

ST_IGNORED, ST_OK, ST_SKIP_NO_LB, ST_REQUEUE_30S, ST_REQUEUE_60S, ST_ERR_RETRY, ST_ERR_NORETRY, ST_PANIC = range(8)
(D_NONE, D_NOT_ELB, D_PARSE_INTERNAL_ALB, D_PARSE_PUBLIC_ALB, D_PARSE_NLB, D_LB_NOT_FOUND, D_LB_DNS_MISMATCH,
 D_TOO_MANY_LISTENERS, D_TOO_MANY_EGS, D_NO_HOSTED_ZONE, D_ACCEL_MANY, D_ACCEL_NONE) = range(12)
EV_CREATED, EV_DELETED = 1, 2

(OP_GA_CREATE_CHAIN, OP_GA_UPDATE_ACCEL, OP_GA_CREATE_LISTENER, OP_GA_UPDATE_LISTENER, OP_GA_CREATE_EG, OP_GA_UPDATE_EG,
 OP_GA_DELETE_CHAIN, OP_R53_CREATE, OP_R53_UPSERT_A, OP_R53_DELETE_RECORD) = range(1, 11)
OP_NAMES = {
    1: "GA_CREATE_CHAIN", 2: "GA_UPDATE_ACCEL", 3: "GA_CREATE_LISTENER", 4: "GA_UPDATE_LISTENER", 5: "GA_CREATE_EG",
    6: "GA_UPDATE_EG", 7: "GA_DELETE_CHAIN", 8: "R53_CREATE", 9: "R53_UPSERT_A", 10: "R53_DELETE_RECORD",
}
CTRL_GA, CTRL_R53 = 0, 1
N_SECTIONS = 4

DV_PROTO_UDP, DV_IP_PRESERVE, DV_IPV4, DV_PORTS_FROM_ANN = 1, 2, 4, 8
DV_GA_ELIGIBLE, DV_GA_MANAGED, DV_R53_ELIGIBLE, DV_R53_ANNOTATED = 16, 32, 64, 128

(TOK_ALB_INTERNAL, TOK_ALB_PUBLIC, TOK_NLB, TOK_NOT_AWS, TOK_PANIC, TOK_ERR_NOT_ELB, TOK_ERR_INTERNAL_ALB,
 TOK_ERR_PUBLIC_ALB, TOK_ERR_NLB) = range(9)

GAR_OK, GAR_E_INVALID, GAR_E_NO_DEVICE, GAR_E_CUDA, GAR_E_STATE, GAR_E_NOMEM = 0, -1, -2, -3, -4, -5

_u8p = C.POINTER(C.c_uint8)
_u32p = C.POINTER(C.c_uint32)
_i32p = C.POINTER(C.c_int32)
_u64p = C.POINTER(C.c_uint64)


class GarObjects(C.Structure):
    _fields_ = [
        ("n_objects", C.c_uint32),
        ("obj_kind", _u8p), ("obj_spec_type", _u8p), ("obj_flags", _u8p),
        ("obj_ns", _u64p), ("obj_name", _u64p), ("obj_ingress_class", _u64p),
        ("obj_ann_begin", _u32p), ("obj_lbi_begin", _u32p), ("obj_port_begin", _u32p),
        ("n_ann", C.c_uint32), ("ann_key", _u64p), ("ann_val", _u64p),
        ("n_lbi", C.c_uint32), ("lbi_hostname", _u64p),
        ("n_ports", C.c_uint32), ("port_number", _i32p), ("port_proto", _u64p),
        ("slab", _u8p), ("slab_len", C.c_uint64),
    ]


class GarActual(C.Structure):
    _fields_ = [
        ("n_lbs", C.c_uint32),
        ("lb_region", _u64p), ("lb_name", _u64p), ("lb_dns", _u64p), ("lb_arn", _u64p), ("lb_state", _u8p),
        ("n_accels", C.c_uint32),
        ("acc_name", _u64p), ("acc_dns", _u64p), ("acc_enabled", _u8p),
        ("acc_tag_begin", _u32p), ("acc_lis_begin", _u32p),
        ("n_tags", C.c_uint32), ("tag_key", _u64p), ("tag_val", _u64p),
        ("n_listeners", C.c_uint32), ("lis_proto", _u8p),
        ("lis_pr_begin", _u32p), ("lis_eg_begin", _u32p),
        ("n_port_ranges", C.c_uint32), ("pr_from", _i32p),
        ("n_egs", C.c_uint32), ("eg_ep_begin", _u32p),
        ("n_endpoints", C.c_uint32), ("ep_id", _u64p),
        ("n_zones", C.c_uint32), ("zone_name", _u64p), ("zone_rec_begin", _u32p),
        ("n_records", C.c_uint32), ("rec_name", _u64p), ("rec_type", _u8p), ("rec_has_alias", _u8p),
        ("rec_alias_dns", _u64p), ("rec_val_begin", _u32p),
        ("n_values", C.c_uint32), ("val_value", _u64p),
        ("slab", _u8p), ("slab_len", C.c_uint64),
    ]


class GarConfig(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("device", C.c_int32), ("cluster_name", C.c_char_p), ("flags", C.c_uint32)]


class GarKeyset(C.Structure):
    _fields_ = [("n_rows", C.c_uint32), ("rows", _u32p), ("n_deleted", C.c_uint32), ("deleted_kind", _u8p), ("deleted_key", C.POINTER(C.c_char_p))]


class GarBindings(C.Structure):
    _fields_ = [
        ("n_bindings", C.c_uint32), ("egb_flags", _u8p), ("egb_ref_kind", _u8p), ("egb_ref_key", _u64p), ("egb_eg_arn", _u64p),
        ("egb_ep_begin", _u32p), ("n_endpoint_ids", C.c_uint32), ("ep_id", _u64p), ("n_known_egs", C.c_uint32), ("known_eg_arn", _u64p),
        ("slab", _u8p), ("slab_len", C.c_uint64),
    ]


EGB_DELETING, EGB_HAS_FINALIZERS, EGB_OBSERVED = 1, 2, 4
(OP_EGB_ADD_FINALIZER, OP_EGB_REMOVE_FINALIZER, OP_EGB_REMOVE_ENDPOINT, OP_EGB_ADD_ENDPOINT, OP_EGB_UPDATE_WEIGHT, OP_EGB_UPDATE_STATUS) = range(11, 17)
ST_REQUEUE_1S = 8
D_REF_NOT_FOUND, D_EG_NOT_FOUND = 12, 13


SHARD_MAX_RANKS, SHARD_META_WORDS, SHARD_HANDLE_BYTES = 8, 40, 96


class GarShard(C.Structure):
    _fields_ = [(k, C.c_uint32) for k in ("rank", "n_ranks", "obj_base", "lb_base", "acc_base", "lis_base", "eg_base", "rec_base", "val_base")]


class GarStageTiming(C.Structure):
    _fields_ = [("name", C.c_char_p), ("ms", C.c_float), ("launches", C.c_uint32), ("bytes", C.c_uint64)]


FLAG_STAGE_TIMING = 1
FLAG_REPREPARE = 2
FLAG_NO_ORPHANS = 4
FLAG_ALLOW_EMPTY_CACHE = 8


class GarOp(C.Structure):
    _fields_ = [("head", C.c_uint32), ("obj", C.c_uint32), ("sub", C.c_uint32), ("a0", C.c_uint32), ("a1", C.c_uint32), ("a2", C.c_uint32)]


OP_DTYPE = np.dtype([("head", "<u4"), ("obj", "<u4"), ("sub", "<u4"), ("a0", "<u4"), ("a1", "<u4"), ("a2", "<u4")])


class GarChangeset(C.Structure):
    _fields_ = [
        ("n_objects", C.c_uint32),
        ("status_ga", _u32p), ("status_r53", _u32p), ("derived", _u32p),
        ("n_ops", C.c_uint64), ("ops", C.POINTER(GarOp)),
        ("section_begin", C.c_uint64 * (N_SECTIONS + 1)),
        ("n_lbi", C.c_uint32), ("tok_code", _u8p), ("tok_name", _u64p), ("tok_region", _u64p),
        ("dport_begin", _u32p), ("n_dports", C.c_uint64), ("dports", _i32p), ("obj_gid", _u32p),
        ("ms_h2d", C.c_float), ("ms_kernels", C.c_float), ("ms_d2h", C.c_float), ("kernel_launches", C.c_uint32),
        ("opaque", C.c_void_p),
    ]


def _np_from(ptr, n, dtype):
    """Copy n elements behind a ctypes pointer into a fresh numpy array (host pointers only)."""
    n = int(n)
    if n == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    addr = C.cast(ptr, C.c_void_p).value
    buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(addr)
    return np.frombuffer(buf, dtype=dtype, count=n).copy()


class ChangeSet:
    """Host copy of a gar_changeset (plain numpy arrays; safe after the C-side object is freed)."""

    def __init__(self, cs: GarChangeset, keyset: bool = False, bindings: bool = False):
        n = cs.n_objects
        self.n_objects = n
        self.status_ga = _np_from(cs.status_ga, n, np.uint32)
        self.status_r53 = _np_from(cs.status_r53, 0 if bindings else n, np.uint32)
        self.derived = _np_from(cs.derived, 0 if bindings else n, np.uint32)
        self.ops = _np_from(cs.ops, cs.n_ops, OP_DTYPE)
        self.section_begin = np.array(list(cs.section_begin), dtype=np.uint64)
        self.tok_code = _np_from(cs.tok_code, cs.n_lbi, np.uint8)
        self.tok_name = _np_from(cs.tok_name, cs.n_lbi, np.uint64)
        self.tok_region = _np_from(cs.tok_region, cs.n_lbi, np.uint64)
        self.dport_begin = _np_from(cs.dport_begin, 0 if keyset else n + 1, np.uint32)
        self.dports = _np_from(cs.dports, cs.n_dports, np.int32)
        self.ms_h2d, self.ms_kernels, self.ms_d2h = cs.ms_h2d, cs.ms_kernels, cs.ms_d2h
        self.kernel_launches = cs.kernel_launches
        self.obj_gid = _np_from(cs.obj_gid, n, np.uint32) if cs.obj_gid else None  # sharded mode only

    ARRAYS = ("status_ga", "status_r53", "derived", "ops", "section_begin", "tok_code", "tok_name", "tok_region", "dport_begin", "dports")

    def diff(self, other: "ChangeSet") -> list[str]:
        """Names of arrays that are not bit-identical."""
        bad = []
        for k in self.ARRAYS:
            a, b = getattr(self, k), getattr(other, k)
            if a.shape != b.shape or not np.array_equal(a, b):
                bad.append(k)
        return bad

    def describe_first_mismatch(self, other: "ChangeSet") -> str:
        for k in self.ARRAYS:
            a, b = getattr(self, k), getattr(other, k)
            if a.shape != b.shape:
                n = min(len(a), len(b))
                idx = next((i for i in range(n) if a[i] != b[i]), n)
                return f"{k}: shape {a.shape} vs {b.shape}; first diff at {idx}: {a[idx] if idx < len(a) else None} vs {b[idx] if idx < len(b) else None}"
            if not np.array_equal(a, b):
                idx = int(np.nonzero(a != b)[0][0])
                return f"{k}[{idx}]: {a[idx]} vs {b[idx]}"
        return "identical"

    def checksum(self) -> int:
        """Order-sensitive 64-bit checksum over every output array (used for big-size parity)."""
        import zlib
        h = 0
        for k in self.ARRAYS:
            a = np.ascontiguousarray(getattr(self, k))
            h = (h * 1000003 + zlib.crc32(a.view(np.uint8).tobytes() if a.size else b"")) & 0xFFFFFFFFFFFFFFFF
        return h


def make_keyset(rows, deleted=()):
    """ctypes gar_keyset from a list of object rows and [(kind, "ns/name"), ...]; keeps its buffers alive on the struct."""
    ks = GarKeyset()
    r = np.ascontiguousarray(np.asarray(list(rows), dtype=np.uint32))
    backing = r if r.size else np.zeros(1, dtype=np.uint32)
    ks.n_rows = int(r.size)
    ks.rows = backing.ctypes.data_as(_u32p)
    kinds = np.ascontiguousarray(np.asarray([k for k, _ in deleted] or [0], dtype=np.uint8))
    keys = (C.c_char_p * max(1, len(deleted)))(*[s.encode() for _, s in deleted])
    ks.n_deleted = len(deleted)
    ks.deleted_kind = kinds.ctypes.data_as(_u8p)
    ks.deleted_key = C.cast(keys, C.POINTER(C.c_char_p))
    ks._keep = (backing, kinds, keys)
    return ks


_lib = None


def load_library(path: os.PathLike | None = None) -> C.CDLL:
    """dlopen libgarecon.so (the CUDA engine).  Raises if it has not been built: there is no fallback."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = Path(path) if path else LIB_PATH
    if not p.exists():
        raise RuntimeError(f"{p} not built - run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
    lib = C.CDLL(str(p))
    lib.gar_engine_create.argtypes = [C.POINTER(GarConfig), C.POINTER(C.c_void_p)]
    lib.gar_engine_create.restype = C.c_int
    lib.gar_engine_destroy.argtypes = [C.c_void_p]
    lib.gar_engine_destroy.restype = None
    for fn in ("gar_snapshot_load", "gar_snapshot_attach_device"):
        getattr(lib, fn).argtypes = [C.c_void_p, C.POINTER(GarObjects), C.POINTER(GarActual)]
        getattr(lib, fn).restype = C.c_int
    for fn in ("gar_diff", "gar_diff_device"):
        getattr(lib, fn).argtypes = [C.c_void_p, C.POINTER(GarChangeset)]
        getattr(lib, fn).restype = C.c_int
    lib.gar_diff_keys.argtypes = [C.c_void_p, C.POINTER(GarKeyset), C.POINTER(GarChangeset)]
    lib.gar_diff_keys.restype = C.c_int
    lib.gar_bindings_diff.argtypes = [C.c_void_p, C.POINTER(GarBindings), C.POINTER(GarChangeset)]
    lib.gar_bindings_diff.restype = C.c_int
    lib.gar_shard_route.argtypes = [C.c_void_p, C.POINTER(GarShard), C.c_int, _u64p, _u64p]
    lib.gar_shard_route.restype = C.c_int
    lib.gar_shard_pack.argtypes = [C.c_void_p, C.c_void_p]
    lib.gar_shard_pack.restype = C.c_int
    lib.gar_shard_unpack.argtypes = [C.c_void_p, C.c_int, C.c_void_p, _u64p]
    lib.gar_shard_unpack.restype = C.c_int
    lib.gar_shard_blob_bytes.argtypes = [_u64p]
    lib.gar_shard_blob_bytes.restype = C.c_uint64
    lib.gar_shard_arena.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.POINTER(C.c_void_p), _u8p, _u64p]
    lib.gar_shard_arena.restype = C.c_int
    lib.gar_shard_open_peers.argtypes = [C.c_void_p, C.c_int, _u8p]
    lib.gar_shard_open_peers.restype = C.c_int
    lib.gar_shard_pack_peers.argtypes = [C.c_void_p, C.c_int, _u64p]
    lib.gar_shard_pack_peers.restype = C.c_int
    lib.gar_changeset_free.argtypes = [C.c_void_p, C.POINTER(GarChangeset)]
    lib.gar_changeset_free.restype = None
    lib.gar_last_error.argtypes = [C.c_void_p]
    lib.gar_last_error.restype = C.c_char_p
    lib.gar_version.argtypes = []
    lib.gar_version.restype = C.c_char_p
    lib.gar_algorithmic_bytes.argtypes = [C.c_void_p, C.POINTER(GarChangeset)]
    lib.gar_algorithmic_bytes.restype = C.c_uint64
    lib.gar_last_stage_timings.argtypes = [C.c_void_p, C.POINTER(GarStageTiming), C.c_uint32]
    lib.gar_last_stage_timings.restype = C.c_uint32
    lib.gar_last_counters.argtypes = [C.c_void_p, _u64p, C.c_uint32]
    lib.gar_last_counters.restype = C.c_uint32
    if path is None:
        _lib = lib
    return lib


EXPORTED_SYMBOLS = (
    "gar_engine_create", "gar_engine_destroy", "gar_snapshot_load", "gar_snapshot_attach_device", "gar_diff",
    "gar_diff_device", "gar_diff_keys", "gar_bindings_diff", "gar_shard_route", "gar_shard_pack", "gar_shard_unpack", "gar_shard_blob_bytes",
    "gar_shard_arena", "gar_shard_open_peers", "gar_shard_pack_peers",
    "gar_changeset_free", "gar_last_error", "gar_version", "gar_algorithmic_bytes",
    "gar_last_stage_timings", "gar_last_counters",
)


class GarError(RuntimeError):
    def __init__(self, rc: int, msg: str):
        super().__init__(f"garecon rc={rc}: {msg}")
        self.rc = rc


class Engine:
    """Thin RAII wrapper over gar_engine_* (one engine per process per device)."""

    def __init__(self, cluster_name: str = "default", device: int = 0, lib: C.CDLL | None = None, stage_timing: bool = False, reprepare: bool = False,
                 orphans: bool = True, allow_empty_cache: bool = False):
        self.lib = lib or load_library()
        self._h = C.c_void_p()
        self._cluster = cluster_name.encode()
        cfg = GarConfig(GAR_ABI_VERSION, device, self._cluster, (FLAG_STAGE_TIMING if stage_timing else 0) | (FLAG_REPREPARE if reprepare else 0)
                        | (0 if orphans else FLAG_NO_ORPHANS) | (FLAG_ALLOW_EMPTY_CACHE if allow_empty_cache else 0))
        rc = self.lib.gar_engine_create(C.byref(cfg), C.byref(self._h))
        if rc != GAR_OK:
            msg = self.lib.gar_last_error(self._h).decode(errors="replace") if self._h else self.lib.gar_last_error(None).decode(errors="replace")
            self._h = C.c_void_p()
            raise GarError(rc, msg)

    def _check(self, rc: int):
        if rc != GAR_OK:
            raise GarError(rc, self.lib.gar_last_error(self._h).decode(errors="replace"))

    def load(self, snap) -> None:
        """snap: anything with .objects (GarObjects) and .actual (GarActual) host structs."""
        self._check(self.lib.gar_snapshot_load(self._h, C.byref(snap.objects), C.byref(snap.actual)))

    def attach_device(self, objects: GarObjects, actual: GarActual) -> None:
        self._check(self.lib.gar_snapshot_attach_device(self._h, C.byref(objects), C.byref(actual)))

    def diff(self) -> ChangeSet:
        cs = GarChangeset()
        self._check(self.lib.gar_diff(self._h, C.byref(cs)))
        try:
            out = ChangeSet(cs)
            out.algorithmic_bytes = int(self.lib.gar_algorithmic_bytes(self._h, C.byref(cs)))
        finally:
            self.lib.gar_changeset_free(self._h, C.byref(cs))
        return out

    def diff_keys(self, rows, deleted=()) -> ChangeSet:
        """Incremental mode: decisions for the object rows `rows` and the deleted keys [(kind, "ns/name"), ...]."""
        ks = make_keyset(rows, deleted)
        cs = GarChangeset()
        self._check(self.lib.gar_diff_keys(self._h, C.byref(ks), C.byref(cs)))
        try:
            cs.n_lbi = 0
            out = ChangeSet(cs, keyset=True)
        finally:
            self.lib.gar_changeset_free(self._h, C.byref(cs))
        return out

    def bindings_diff(self, bindings) -> ChangeSet:
        """EndpointGroupBinding set-diff against the loaded snapshot; `bindings` has a .struct (GarBindings)."""
        cs = GarChangeset()
        self._check(self.lib.gar_bindings_diff(self._h, C.byref(bindings.struct), C.byref(cs)))
        try:
            out = ChangeSet(cs, keyset=True, bindings=True)
        finally:
            self.lib.gar_changeset_free(self._h, C.byref(cs))
        return out

    # ---- sharded mode (include/garecon.h "sharded mode"): the caller moves the blobs between the calls
    def shard_route(self, shard: GarShard, rnd: int):
        """-> (meta [n_ranks, SHARD_META_WORDS] uint64, send_bytes [n_ranks] uint64) of this rank's outgoing blobs."""
        g = int(shard.n_ranks)
        meta = np.zeros((g, SHARD_META_WORDS), dtype=np.uint64)
        nbytes = np.zeros(g, dtype=np.uint64)
        self._check(self.lib.gar_shard_route(self._h, C.byref(shard), rnd, meta.ctypes.data_as(_u64p), nbytes.ctypes.data_as(_u64p)))
        return meta, nbytes

    def shard_pack(self, send_ptr: int) -> None:
        self._check(self.lib.gar_shard_pack(self._h, C.c_void_p(send_ptr)))

    def shard_unpack(self, rnd: int, recv_ptr: int, recv_meta: np.ndarray) -> None:
        m = np.ascontiguousarray(recv_meta, dtype=np.uint64)
        self._check(self.lib.gar_shard_unpack(self._h, rnd, C.c_void_p(recv_ptr), m.ctypes.data_as(_u64p)))

    # peer-memory exchange (include/garecon.h): pack kernels store straight into the other ranks' receive arenas
    def shard_arena(self, rnd: int, need_bytes: int):
        """-> (arena device pointer, handle bytes [SHARD_HANDLE_BYTES] uint8, capacity in bytes) of this rank's receive arena of
        round `rnd`; need_bytes = 0 asks for the arena as it stands."""
        ptr = C.c_void_p()
        cap = C.c_uint64()
        handle = np.zeros(SHARD_HANDLE_BYTES, dtype=np.uint8)
        self._check(self.lib.gar_shard_arena(self._h, rnd, int(need_bytes), C.byref(ptr), handle.ctypes.data_as(_u8p), C.byref(cap)))
        return int(ptr.value), handle, int(cap.value)

    def shard_open_peers(self, rnd: int, handles: np.ndarray) -> None:
        h = np.ascontiguousarray(handles, dtype=np.uint8)
        self._check(self.lib.gar_shard_open_peers(self._h, rnd, h.ctypes.data_as(_u8p)))

    def shard_pack_peers(self, rnd: int, all_meta: np.ndarray) -> None:
        m = np.ascontiguousarray(all_meta, dtype=np.uint64)
        self._check(self.lib.gar_shard_pack_peers(self._h, rnd, m.ctypes.data_as(_u64p)))

    def blob_bytes(self, meta_row: np.ndarray) -> int:
        m = np.ascontiguousarray(meta_row, dtype=np.uint64)
        return int(self.lib.gar_shard_blob_bytes(m.ctypes.data_as(_u64p)))

    def diff_raw(self) -> dict:
        """gar_diff + gar_changeset_free without copying the arrays into numpy: what a C / cgo caller pays.
        Returns counts and timings only."""
        cs = GarChangeset()
        self._check(self.lib.gar_diff(self._h, C.byref(cs)))
        out = {"n_ops": int(cs.n_ops), "n_dports": int(cs.n_dports), "ms_h2d": cs.ms_h2d, "ms_kernels": cs.ms_kernels, "ms_d2h": cs.ms_d2h,
               "kernel_launches": int(cs.kernel_launches), "first_status": int(cs.status_ga[0]) if cs.n_objects else 0}
        self.lib.gar_changeset_free(self._h, C.byref(cs))
        return out

    def diff_device(self) -> GarChangeset:
        """Kernels only; result stays on the device.  Returns the raw struct (counts + timings valid)."""
        cs = GarChangeset()
        self._check(self.lib.gar_diff_device(self._h, C.byref(cs)))
        return cs

    def stage_timings(self) -> list[tuple[str, float, int]]:
        """(name, ms, launches) per stage of the last diff (engine created with stage_timing=True)."""
        arr = (GarStageTiming * 128)()
        n = self.lib.gar_last_stage_timings(self._h, arr, 128)
        return [(arr[i].name.decode(), float(arr[i].ms), int(arr[i].launches)) for i in range(min(n, 128))]

    def counters(self) -> dict:
        """Exact sizes of the intermediate relations of the last diff (include/garecon.h GAR_CTR_*)."""
        arr = (C.c_uint64 * 8)()
        n = self.lib.gar_last_counters(self._h, arr, 8)
        names = ("r53_pairs", "dports")
        return {names[i]: int(arr[i]) for i in range(min(n, len(names)))}

    def algorithmic_bytes(self, cs: GarChangeset) -> int:
        return int(self.lib.gar_algorithmic_bytes(self._h, C.byref(cs)))

    def close(self):
        if self._h:
            self.lib.gar_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
