"""Object deltas against a reload: one JSON line on stdout.

  python profiles/delta_bench.py [--config 3] [--objects 1000000] [--batches 6] [--warmup 2] [--churn 0.01] [--seed 11]

Workload: bench.py's timed snapshot (BASELINE configs[2] at 10^6 objects, column-major slabs, rank 0's seed), then batches of
informer-like churn from deltas.churn (updates that change an lbIngress hostname / route53-hostname / listen-ports annotation,
0.05 % adds with fresh keys, 0.05 % deletes), deterministic from --seed.  Per batch:
  delta     gar_snapshot_apply_objects(batch) on the resident, prepared snapshot, then gar_diff_keys of the touched keys
            (the first diff after the delta: it rebuilds the object side), then the first full diff (orphan values too);
  reload    gar_snapshot_load of the equivalent table (its object columns and both slabs pinned like bench.py's e2e arm; the
            AWS columns are the timed snapshot's, pinned as well) + the same gar_diff_keys, on a second engine.
Host clock around calls that synchronise; the first --warmup batches are not timed; medians.  `equal`: after the last batch
the full diff of the delta-fed engine equals that of a fresh load of the equivalent table — deltas.ColumnMirror lays its slab
out like the resident one, so every array, tok_name / tok_region included, is compared bit for bit.  Like bench.py it runs
on the tree as __graft_entry__.build() left it and writes nothing into it.
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
    ap.add_argument("--seed", type=int, default=11)
    args = ap.parse_args()
    if args.batches <= args.warmup:
        ap.error("--batches must exceed --warmup")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("delta_bench.py needs a CUDA device: the engine has no CPU path")
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
    mirror = deltas.ColumnMirror(tables.columns(snap.objects, tables.OBJ_TABLES))
    a_cols = tables.columns(snap.actual, tables.ACT_TABLES)
    rng = np.random.default_rng(args.seed)
    eng = pkg.Engine(cluster_name=snap.cluster)
    beng = pkg.Engine(cluster_name=snap.cluster)
    cs = abi.GarChangeset()

    def keys_diff(e, ks):
        e._check(e.lib.gar_diff_keys(e._h, C.byref(ks), C.byref(cs)))
        e.lib.gar_changeset_free(e._h, C.byref(cs))

    def full_diff(e):
        e._check(e.lib.gar_diff(e._h, C.byref(cs)))
        e.lib.gar_changeset_free(e._h, C.byref(cs))

    eng.load(snap)
    full_diff(eng)  # prepared: digests and indexes resident
    rec = {k: [] for k in ("ms_apply", "ms_diff_keys", "ms_full_after", "ms_load", "ms_load_diff_keys", "upsert_bytes", "upserts", "deletes")}
    msnap = None
    for b in range(args.batches):
        up, deleted = deltas.churn(mirror, rng, frac=args.churn, serial=b)
        keep, uobj = deltas.objects_struct(up)
        nu = int(uobj.n_objects)
        ubytes = (int(uobj.slab_len) + nu * (3 + 3 * 8) + 3 * 4 * (nu + 1) + 16 * int(uobj.n_ann) + 8 * int(uobj.n_lbi) + 12 * int(uobj.n_ports)
                  + sum(len(k) + 1 for _, k in deleted))
        t0 = time.perf_counter()
        res = eng.apply_objects(uobj, deleted)
        t1 = time.perf_counter()
        ks = abi.make_keyset(res.upsert_row.tolist(), deleted)
        keys_diff(eng, ks)
        t2 = time.perf_counter()
        full_diff(eng)
        t3 = time.perf_counter()
        rows, _, _ = mirror.apply(up, deleted)
        if not np.array_equal(rows, res.upsert_row):
            raise RuntimeError("delta rows differ from the table-level mirror")
        del msnap
        msnap = mirror.snapshot(a_cols)
        # the fresh object columns and both slabs; the AWS columns are views of the timed snapshot's arrays, which are
        # registered already (registering a range twice is an error)
        rt, addrs = torch.cuda.cudart(), []
        arrays = bench._table_arrays(abi, msnap.objects, msnap.actual)
        for ptr, cnt, sz in arrays[:15] + arrays[-1:]:
            addr = C.cast(ptr, C.c_void_p).value
            if addr and cnt and int(rt.cudaHostRegister(addr, int(cnt) * sz, 0)) == 0:
                addrs.append(addr)
        t4 = time.perf_counter()
        beng.load(msnap)
        t5 = time.perf_counter()
        keys_diff(beng, ks)
        t6 = time.perf_counter()
        bench._unpin(torch, addrs)
        if b < args.warmup:
            continue
        for k, v in (("ms_apply", t1 - t0), ("ms_diff_keys", t2 - t1), ("ms_full_after", t3 - t2), ("ms_load", t5 - t4), ("ms_load_diff_keys", t6 - t5)):
            rec[k].append(v * 1e3)
        rec["upsert_bytes"].append(ubytes)
        rec["upserts"].append(nu)
        rec["deletes"].append(len(deleted))
    got, want = eng.diff(), beng.diff()
    bad = got.diff(want)
    out = {"device": bench._device_info(torch.cuda.current_device()),
           "config": {"workload": f"BASELINE configs index {args.config}, {args.objects} objects, column-major slabs", "seed": int(cfg.seed),
                      "churn": args.churn, "churn_seed": args.seed}}
    out.update({k: round(float(np.median(v)), 3) for k, v in rec.items() if k.startswith("ms_")})
    out.update({"batches_timed": args.batches - args.warmup, "upserts_per_batch": int(np.median(rec["upserts"])),
                "deletes_per_batch": int(np.median(rec["deletes"])), "upsert_h2d_bytes": int(np.median(rec["upsert_bytes"])),
                "load_h2d_bytes": int(sum(int(c) * s for (_, c, s) in bench._table_arrays(abi, msnap.objects, msnap.actual))),
                "resident_slab_bytes": int(res.slab_len), "equal": not bad})
    out["ms_apply_plus_diff_keys"] = round(out["ms_apply"] + out["ms_diff_keys"], 3)
    out["ms_load_plus_diff_keys"] = round(out["ms_load"] + out["ms_load_diff_keys"], 3)
    out["apply_beats_load"] = out["ms_apply_plus_diff_keys"] < out["ms_load_plus_diff_keys"]
    if bad:
        out["mismatch"] = {"arrays": bad, "first": got.describe_first_mismatch(want)}
    eng.close()
    beng.close()
    bench._unpin(torch, snap_pins)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
