"""AWS deltas against a reload: one JSON line on stdout.

  python profiles/actual_delta_bench.py [--config 3] [--objects 1000000] [--batches 6] [--warmup 2] [--churn 0.01] [--seed 17]

Workload: bench.py's timed snapshot (BASELINE configs[2] at 10^6 objects, column-major slabs, rank 0's seed), then re-list
batches from deltas.aws_churn (LB state flips, appends and deletes; rewritten, appended and deleted accelerator subtrees; the
record lists of four zones replaced), deterministic from --seed.  A fixed 1 % batch of object rows is the gar_diff_keys batch.
Per batch:
  delta     gar_snapshot_apply_actual(batch) on the resident snapshot, then gar_diff_keys of the key batch (the first diff after
            the delta: it re-prepares the whole snapshot), then the first full diff;
  reload    gar_snapshot_load of the equivalent tables (pinned like bench.py's e2e arm) + the same gar_diff_keys, on a second
            engine.
Host clock around calls that synchronise; the first --warmup batches are not timed; medians.  `equal`: after the last batch the
full diff of the delta-fed engine equals that of a fresh load of the mirrored tables (deltas.ActualMirror).  Like bench.py it
runs on the tree as __graft_entry__.build() left it and writes nothing into it.
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

import bench  # noqa: E402  (table pinning, device info: the same helpers as the e2e arm)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--objects", type=int, default=1_000_000)
    ap.add_argument("--batches", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--churn", type=float, default=0.01)
    ap.add_argument("--seed", type=int, default=17)
    args = ap.parse_args()
    if args.batches <= args.warmup:
        ap.error("--batches must exceed --warmup")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("actual_delta_bench.py needs a CUDA device: the engine has no CPU path")
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
    _, snap_pins = bench._pin_host_tables(torch, abi, snap.objects, snap.actual)
    mirror = deltas.ActualMirror(tables.columns(snap.actual, tables.ACT_TABLES))
    o_cols = tables.columns(snap.objects, tables.OBJ_TABLES)
    rng = np.random.default_rng(args.seed)
    n = int(snap.objects.n_objects)
    key_rows = np.sort(np.random.default_rng(args.seed + 1).choice(n, size=max(1, n // 100), replace=False)).tolist()
    ks = abi.make_keyset(key_rows)
    eng = pkg.Engine(cluster_name=snap.cluster)
    beng = pkg.Engine(cluster_name=snap.cluster)
    cs = abi.GarChangeset()

    def keys_diff(e):
        e._check(e.lib.gar_diff_keys(e._h, C.byref(ks), C.byref(cs)))
        e.lib.gar_changeset_free(e._h, C.byref(cs))

    def full_diff(e):
        e._check(e.lib.gar_diff(e._h, C.byref(cs)))
        e.lib.gar_changeset_free(e._h, C.byref(cs))

    eng.load(snap)
    full_diff(eng)  # prepared, as a worker's engine is between batches
    rec = {k: [] for k in ("ms_apply", "ms_diff_keys", "ms_full_after", "ms_load", "ms_load_diff_keys", "delta_bytes")}
    msnap = None
    for b in range(args.batches):
        d = deltas.aws_churn(mirror, rng, frac=args.churn)
        keep, rows = deltas.actual_struct(d["rows"])
        dbytes = sum(int(c) * s for (_, c, s) in bench._table_arrays(abi, keep.objects, rows)) + 4 * sum(
            len(d[k]) for k in ("lb_target", "acc_target", "zone_target", "lb_deleted", "acc_deleted"))
        t0 = time.perf_counter()
        res = eng.apply_actual(rows, d["lb_target"], d["acc_target"], d["zone_target"], d["lb_deleted"], d["acc_deleted"])
        t1 = time.perf_counter()
        keys_diff(eng)
        t2 = time.perf_counter()
        full_diff(eng)
        t3 = time.perf_counter()
        want = mirror.apply(**d)
        if tuple(res) != tuple(want[k] for k in abi.ActualDeltaResult.FIELDS):
            raise RuntimeError(f"delta result {tuple(res)} differs from the table-level mirror {want}")
        del msnap
        msnap = mirror.snapshot(o_cols)
        # the fresh AWS columns and both slabs; the object columns are views of the timed snapshot's arrays, which are
        # registered already (registering a range twice is an error)
        rt, addrs = torch.cuda.cudart(), []
        arrays = bench._table_arrays(abi, msnap.objects, msnap.actual)
        for ptr, cnt, sz in arrays[14:]:
            addr = C.cast(ptr, C.c_void_p).value
            if addr and cnt and int(rt.cudaHostRegister(addr, int(cnt) * sz, 0)) == 0:
                addrs.append(addr)
        t4 = time.perf_counter()
        beng.load(msnap)
        t5 = time.perf_counter()
        keys_diff(beng)
        t6 = time.perf_counter()
        bench._unpin(torch, addrs)
        if b < args.warmup:
            continue
        for k, v in (("ms_apply", t1 - t0), ("ms_diff_keys", t2 - t1), ("ms_full_after", t3 - t2), ("ms_load", t5 - t4), ("ms_load_diff_keys", t6 - t5)):
            rec[k].append(v * 1e3)
        rec["delta_bytes"].append(dbytes)
    got, want = eng.diff(), beng.diff()
    bad = got.diff(want)
    out = {"device": bench._device_info(torch.cuda.current_device()),
           "config": {"workload": f"BASELINE configs index {args.config}, {args.objects} objects, column-major slabs", "seed": int(cfg.seed),
                      "churn": args.churn, "churn_seed": args.seed, "diff_keys_rows": len(key_rows)}}
    out.update({k: round(float(np.median(v)), 3) for k, v in rec.items() if k.startswith("ms_")})
    out.update({"batches_timed": args.batches - args.warmup, "delta_h2d_bytes": int(np.median(rec["delta_bytes"])),
                "load_h2d_bytes": int(sum(int(c) * s for (_, c, s) in bench._table_arrays(abi, msnap.objects, msnap.actual))),
                "resident_aws_slab_bytes": int(res.slab_len), "equal": not bad})
    out["ms_apply_plus_diff_keys"] = round(out["ms_apply"] + out["ms_diff_keys"], 3)
    out["ms_load_plus_diff_keys"] = round(out["ms_load"] + out["ms_load_diff_keys"], 3)
    if bad:
        out["mismatch"] = {"arrays": bad, "first": got.describe_first_mismatch(want)}
    eng.close()
    beng.close()
    bench._unpin(torch, snap_pins)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
