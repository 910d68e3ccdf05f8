"""Zone deltas against a reload: one JSON line on stdout.

  python profiles/zone_delta_bench.py [--config 3] [--objects 1000000] [--reps 5] [--seed 19]

Workload: bench.py's timed snapshot (BASELINE configs[2] at 10^6 objects, column-major slabs, rank 0's seed).  Three arms, each
run --reps times from the loaded, prepared snapshot (the same delta every time, deterministic from --seed):
  add_empty   one new hosted zone without records (deltas.zone_churn, n_add=1, rec_frac=0);
  add_10      ten new zones whose records total ~1 % of all records: a subzone of the busiest zone, a duplicate name listed in
              front of its namesake, eight fresh names (deltas.zone_churn, n_add=10, rec_frac=0.01);
  delete_10   the ten zones with the most records deleted, with their record sets (deltas.largest_zones_deleted).
Per repetition:
  delta     gar_snapshot_apply_zones on the resident snapshot, then gar_diff_keys of a fixed 1 % key batch (the first diff after
            the delta: it re-prepares the whole snapshot), then the first full diff;
  reload    gar_snapshot_load of the resulting tables (pinned like bench.py's e2e arm) + the same gar_diff_keys, on a second
            engine.
Host clock around calls that synchronise; medians with min-max.  `equal`: after every repetition the full diff of the
delta-fed engine equals that of the reloaded one.  Like bench.py it runs on the tree as __graft_entry__.build() left it and
writes nothing into it.
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=19)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("zone_delta_bench.py needs a CUDA device: the engine has no CPU path")
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
    a_cols = tables.columns(snap.actual, tables.ACT_TABLES)
    o_cols = tables.columns(snap.objects, tables.OBJ_TABLES)
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

    arms = {
        "add_empty": lambda m, rng: deltas.zone_churn(m, rng, n_add=1, rec_frac=0.0),
        "add_10": lambda m, rng: deltas.zone_churn(m, rng, n_add=10, rec_frac=0.01),
        "delete_10": lambda m, rng: deltas.largest_zones_deleted(m, 10),
    }
    out = {"device": bench._device_info(torch.cuda.current_device()),
           "config": {"workload": f"BASELINE configs index {args.config}, {args.objects} objects, column-major slabs", "seed": int(cfg.seed),
                      "zone_seed": args.seed, "reps": args.reps, "diff_keys_rows": len(key_rows),
                      "resident": {"n_zones": int(snap.actual.n_zones), "n_records": int(snap.actual.n_records), "n_values": int(snap.actual.n_values)}}}
    equal = True
    for ai, (name, make) in enumerate(arms.items()):
        rec = {k: [] for k in ("ms_apply", "ms_diff_keys", "ms_full_after", "ms_load", "ms_load_diff_keys")}
        for rep in range(args.reps):
            eng.load(snap)
            full_diff(eng)  # prepared, as a worker's engine is between batches
            mirror = deltas.ActualMirror(a_cols)
            d = make(mirror, np.random.default_rng(args.seed + ai))
            keep, added = deltas.actual_struct(d["added"]) if d["added"] is not None else (None, None)
            dbytes = 4 * (len(d["added_at"]) + len(d["deleted"]))
            if added is not None:
                dbytes += sum(int(c) * s for (_, c, s) in bench._table_arrays(abi, keep.objects, added))
            t0 = time.perf_counter()
            res = eng.apply_zones(added, d["added_at"], d["deleted"])
            t1 = time.perf_counter()
            keys_diff(eng)
            t2 = time.perf_counter()
            full_diff(eng)
            t3 = time.perf_counter()
            want = mirror.apply_zones(**d)
            if tuple(res) != tuple(want[k] for k in abi.ZoneDeltaResult.FIELDS):
                raise RuntimeError(f"{name}: delta result {tuple(res)} differs from the table-level mirror {want}")
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
            got, ref = eng.diff(), beng.diff()
            bad = got.diff(ref)
            if bad:
                equal = False
                out.setdefault("mismatch", {})[name] = {"arrays": bad, "first": got.describe_first_mismatch(ref)}
            for k, v in (("ms_apply", t1 - t0), ("ms_diff_keys", t2 - t1), ("ms_full_after", t3 - t2), ("ms_load", t5 - t4), ("ms_load_diff_keys", t6 - t5)):
                rec[k].append(v * 1e3)
            rec.setdefault("ms_apply_plus_diff_keys", []).append((t2 - t0) * 1e3)
            rec.setdefault("ms_load_plus_diff_keys", []).append((t6 - t4) * 1e3)
            load_bytes = int(sum(int(c) * s for (_, c, s) in arrays))
            del msnap, keep, added
        arm = {k: {"median": round(float(np.median(v)), 3), "min": round(float(np.min(v)), 3), "max": round(float(np.max(v)), 3)} for k, v in rec.items()}
        arm.update({"delta_h2d_bytes": int(dbytes), "load_h2d_bytes": load_bytes, "after": {k: int(getattr(res, k)) for k in ("n_zones", "n_records", "n_values")},
                    "resident_aws_slab_bytes": int(res.slab_len)})
        out[name] = arm
    out["equal"] = equal
    eng.close()
    beng.close()
    bench._unpin(torch, snap_pins)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
