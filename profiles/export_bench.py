"""Export of the resident snapshot to host memory (gar_snapshot_export) against the plain copy it aims at: one JSON line on stdout.

  python profiles/export_bench.py [--config 3] [--objects 1000000] [--churn 0.1] [--batches 4] [--reps 5] [--seed 17]
                                  [--baseline-lib PATH]

Workload: profiles/compact_bench.py's: bench.py's timed snapshot (BASELINE configs[2] at 10^6 objects, column-major slabs, rank
0's seed) after --batches batches of deltas.churn and deltas.aws_churn (deterministic from --seed) on the engine, so its slabs
hold dead strings.  Reported, medians over --reps repetitions with min / max, host clock around calls that end in a device
synchronise:
  export      gar_snapshot_export of the object group, the AWS group and both, into pinned memory (torch pin_memory) and into
              pageable memory (numpy), size query included (Engine.export); bytes = the buffer bytes used;
  d2h         a plain cudaMemcpy device -> pinned host of the same byte count (torch copy_ + synchronize): the floor the
              pipelined gather aims at; export / d2h is reported;
  restore     gar_snapshot_load of the exported tables (pinned) into a second engine;
  compact     gar_snapshot_compact of each group on a fresh load of the grown tables, this build and, with --baseline-lib, the
              library of the previous commit, alternating;
  equal       the engine loaded from the export gives the full diff of the source engine: tok_name / tok_region as the strings
              they name, every other array bit for bit.
Like bench.py it runs on the tree as __graft_entry__.build() left it and writes nothing into it.
"""
import argparse
import ctypes as C
import importlib
import json
import sys
import time
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402

import bench  # noqa: E402
from compact_bench import stats, tok_strings  # noqa: E402

OBJ, ACT, BOTH = 1, 2, 3


def baseline_lib(path, abi):
    """The few entry points a compaction needs, from a library that may predate gar_snapshot_export."""
    lib = C.CDLL(str(path))
    lib.gar_engine_create.argtypes = [C.POINTER(abi.GarConfig), C.POINTER(C.c_void_p)]
    lib.gar_engine_destroy.argtypes = [C.c_void_p]
    lib.gar_engine_destroy.restype = None
    lib.gar_snapshot_load.argtypes = [C.c_void_p, C.POINTER(abi.GarObjects), C.POINTER(abi.GarActual)]
    lib.gar_snapshot_compact.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.GarCompactResult)]
    lib.gar_last_error.argtypes = [C.c_void_p]
    lib.gar_last_error.restype = C.c_char_p
    return lib


def timed(fn, reps):
    fn()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ms.append((time.perf_counter() - t0) * 1e3)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--objects", type=int, default=1_000_000)
    ap.add_argument("--churn", type=float, default=0.1)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=17)
    ap.add_argument("--baseline-lib", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("export_bench.py needs a CUDA device: the engine has no CPU path")
    bench._require_built()
    pkg = importlib.import_module("aws-global-accelerator-controller_b200")
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    ranks = importlib.import_module("aws-global-accelerator-controller_b200.ranks")
    deltas = importlib.import_module("aws-global-accelerator-controller_b200.deltas")
    abi, tables = pkg.abi, pkg.tables

    cfg = synth.preset(args.config, args.objects)
    cfg.seed = ranks.rank_seed(cfg.seed, 0)
    cfg.layout = 1
    snap = synth.SynthSnapshot(cfg)
    om = deltas.ColumnMirror(tables.columns(snap.objects, tables.OBJ_TABLES))
    am = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    loaded = (om.slab_len, am.slab_len)
    rng = np.random.default_rng(args.seed)
    eng = pkg.Engine(cluster_name=snap.cluster)
    eng.load(snap)
    zones = max(4, len(am.cur["zone_name"]) // 8)
    for b in range(args.batches):
        up, deleted = deltas.churn(om, rng, frac=args.churn, serial=b)
        keep, uobj = deltas.objects_struct(up)
        eng.apply_objects(uobj, deleted)
        om.apply(up, deleted)
        d = deltas.aws_churn(am, rng, frac=args.churn, max_zones=zones)
        keep2, rows = deltas.actual_struct(d["rows"])
        eng.apply_actual(rows, d["lb_target"], d["acc_target"], d["zone_target"], d["lb_deleted"], d["acc_deleted"])
        am.apply(**d)
    grown = tables.from_columns(om.cur, am.cur)
    out = {"device": bench._device_info(torch.cuda.current_device()),
           "config": {"workload": f"BASELINE configs index {args.config}, {args.objects} objects, column-major slabs", "seed": int(cfg.seed),
                      "churn": args.churn, "churn_seed": args.seed, "batches": args.batches, "reps": args.reps},
           "slab_growth": {"objects": round(om.slab_len / loaded[0], 3), "actual": round(am.slab_len / loaded[1], 3)}}

    # export of each group and of both, pinned and pageable, against a plain D2H of the same bytes
    need = eng.export_size(BOTH)
    total = ((int(need.obj_bytes) + 15) & ~15) + int(need.act_bytes)
    pinned = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    pageable = np.empty(total, dtype=np.uint8)
    dev = torch.empty(total, dtype=torch.uint8, device="cuda")
    dev.fill_(1)
    res = {}
    for name, g in (("objects", OBJ), ("actual", ACT), ("both", BOTH)):
        sz = eng.export_size(g)
        nbytes = int(sz.obj_bytes) + int(sz.act_bytes)
        r = {"bytes": nbytes}
        for kind, buf in (("pinned", pinned.numpy()), ("pageable", pageable)):
            r[f"ms_{kind}"] = stats(timed(lambda: eng.export(g, buf), args.reps))

        def d2h():
            pinned[:nbytes].copy_(dev[:nbytes], non_blocking=True)
            torch.cuda.synchronize()
        r["ms_plain_d2h_pinned"] = stats(timed(d2h, args.reps))
        r["export_pinned_over_d2h"] = round(r["ms_pinned"]["median"] / r["ms_plain_d2h_pinned"]["median"], 3)
        r["d2h_GBps"] = round(nbytes / (r["ms_plain_d2h_pinned"]["median"] * 1e-3) / 1e9, 1)
        res[name] = r
    out["export"] = res

    # the restore, and the answers of the restored engine
    x = eng.export(BOTH, pinned.numpy())
    e2 = pkg.Engine(cluster_name=snap.cluster)
    out["ms_restore_load_pinned"] = stats(timed(lambda: e2.load(x), args.reps))
    want, got = eng.diff(), e2.diff()
    src_slab = eng.read_slab(OBJ, 0, om.slab_len)
    x_slab = np.array(np.ctypeslib.as_array(x.objects.slab, shape=(max(1, x.objects.slab_len),))[:x.objects.slab_len])
    bad = []
    for name in want.ARRAYS:
        a, b = getattr(want, name), getattr(got, name)
        if name in ("tok_name", "tok_region"):
            (la, sa), (lb, sb) = tok_strings(a, src_slab), tok_strings(b, x_slab)
            same = np.array_equal(la, lb) and np.array_equal(sa, sb)
        else:
            same = a.shape == b.shape and np.array_equal(a, b)
        if not same:
            bad.append(name)
    om.compact()
    am.compact()
    layout_ok = all(np.array_equal(tables.columns(x.objects, tables.OBJ_TABLES)[k], om.cur[k]) for k in om.cur) and \
        all(np.array_equal(tables.columns(x.actual, tables.ACT_TABLES)[k], am.cur[k]) for k in am.cur)
    out["equal"] = not bad and layout_ok
    if bad or not layout_ok:
        out["mismatch"] = bad + ([] if layout_ok else ["layout"])
    e2.close()
    eng.close()

    # the compaction, this build against the baseline library, alternating
    arms = {"this": pkg.Engine(cluster_name=snap.cluster)}
    if args.baseline_lib:
        arms["baseline"] = pkg.Engine(cluster_name=snap.cluster, lib=baseline_lib(args.baseline_lib, abi))
    cms = {k: {OBJ: [], ACT: []} for k in arms}
    for rep in range(args.reps + 1):
        for k, e in arms.items():
            e.load(grown)
            for g in (OBJ, ACT):
                t0 = time.perf_counter()
                e.compact(g)
                if rep:
                    cms[k][g].append((time.perf_counter() - t0) * 1e3)
    out["ms_compact"] = {k: {"objects": stats(v[OBJ]), "actual": stats(v[ACT])} for k, v in cms.items()}
    for e in arms.values():
        e.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
