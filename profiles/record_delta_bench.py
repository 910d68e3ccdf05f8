"""The refresh loop of a delta-fed worker at zone and at record granularity, alternated in one process: one JSON line on stdout.

  python profiles/record_delta_bench.py [--config 2] [--objects 1000000] [--rows 10000] [--deleted 100] [--reps 11] [--seed 17]

Workload: profiles/read_set_bench.py's (bench.py's timed snapshot, BASELINE configs[2] at 10^6 objects; --rows object rows drawn
with --seed plus the keys of --deleted other objects passed as deleted keys).  The two loops, alternated rep by rep, each with
the rows re-described unchanged (taken from the loaded tables outside the timed window: a worker gets them from AWS), so the
resident tables stay what they were:
  zone     gar_read_set -> gar_snapshot_apply_actual(LBs, accelerators, whole zone record lists) -> gar_diff_keys;
  record   gar_read_set -> gar_read_records -> gar_snapshot_apply_actual(LBs, accelerators) -> gar_snapshot_apply_records(the
           record rows, each replaced by itself) -> gar_diff_keys.
Reported, medians over --reps with min and max, host clock around calls that synchronise: each loop, each apply call on its own,
gar_read_records, the set sizes and the bytes each delta carries to the device (columns + slab).  `equal`: every loop's change set
equals the plain gar_diff_keys' on the loaded snapshot.  Like bench.py it runs on the tree as __graft_entry__.build() left it
and writes nothing into it.
"""
import argparse
import importlib
import json
import random
import statistics
import sys
import time
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402

import bench  # noqa: E402  (device info and the built-library check: the same helpers as bench.py)


def stats(ts):
    ms = [t * 1e3 for t in ts]
    return {"median_ms": round(statistics.median(ms), 4), "min_ms": round(min(ms), 4), "max_ms": round(max(ms), 4)}


def delta_bytes(cols):
    """Bytes of a delta's columns and slab: what the apply call copies to the device."""
    return int(sum(np.asarray(v).nbytes for v in cols.values()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2)
    ap.add_argument("--objects", type=int, default=1_000_000)
    ap.add_argument("--rows", type=int, default=10_000)
    ap.add_argument("--deleted", type=int, default=100)
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--seed", type=int, default=17)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("record_delta_bench.py needs a CUDA device: the engine has no CPU path")
    bench._require_built()
    pkg = importlib.import_module("aws-global-accelerator-controller_b200")
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    ranks = importlib.import_module("aws-global-accelerator-controller_b200.ranks")
    deltas = importlib.import_module("aws-global-accelerator-controller_b200.deltas")
    tables = pkg.tables

    cfg = synth.preset(args.config, args.objects)
    cfg.seed = ranks.rank_seed(cfg.seed, 0)
    cfg.layout = 1
    snap = synth.SynthSnapshot(cfg)
    rng = random.Random(args.seed)
    n = int(snap.objects.n_objects)
    cols = tables.columns(snap.objects, tables.OBJ_TABLES)
    slab = np.ctypeslib.as_array(snap.objects.slab, shape=(int(snap.objects.slab_len),))

    def key(i):
        ns, nm = int(cols["obj_ns"][i]), int(cols["obj_name"][i])
        off, ln = ns & ((1 << 40) - 1), (ns >> 40) + 1 + (nm >> 40)
        return int(cols["obj_kind"][i]), bytes(slab[off:off + ln]).decode()

    picks = rng.sample(range(n), args.rows + args.deleted)
    rows, gone = picks[:args.rows], picks[args.rows:]
    deleted = [key(i) for i in gone]
    act = tables.columns(snap.actual, tables.ACT_TABLES)

    with pkg.Engine(cluster_name="default", device=0) as e:
        e.load(snap)
        base = e.diff_keys(rows, deleted)  # prepares the snapshot and builds ix_owner / ix_val
        rs = e.read_set(rows, deleted)
        rr = e.read_records(rows, deleted)
        zone_cols = deltas.compact_actual(deltas.actual_rows(act, rs.lb_rows, rs.acc_rows, rs.zone_rows))
        aws_cols = deltas.compact_actual(deltas.actual_rows(act, rs.lb_rows, rs.acc_rows))
        rec = deltas.record_redescribe(act, rr)
        keep = [deltas.actual_struct(c) for c in (zone_cols, aws_cols, rec["rows"])]
        zone_delta, aws_delta, rec_delta = (k[1] for k in keep)
        t = {k: [] for k in ("zone_loop", "zone_apply_actual", "record_loop", "read_records", "record_apply_actual", "apply_records")}
        equal = True
        for _ in range(args.reps):
            t0 = time.perf_counter()
            rs = e.read_set(rows, deleted)
            t1 = time.perf_counter()
            e.apply_actual(zone_delta, rs.lb_rows, rs.acc_rows, rs.zone_rows)
            t2 = time.perf_counter()
            cs = e.diff_keys(rows, deleted)
            t3 = time.perf_counter()
            t["zone_loop"].append(t3 - t0)
            t["zone_apply_actual"].append(t2 - t1)
            equal = equal and cs.diff(base) == []

            t0 = time.perf_counter()
            rs = e.read_set(rows, deleted)
            t1 = time.perf_counter()
            rr = e.read_records(rows, deleted)
            t2 = time.perf_counter()
            e.apply_actual(aws_delta, rs.lb_rows, rs.acc_rows)
            t3 = time.perf_counter()
            e.apply_records(rec_delta, rec["zone_target"], rr, rr)
            t4 = time.perf_counter()
            cs = e.diff_keys(rows, deleted)
            t5 = time.perf_counter()
            t["record_loop"].append(t5 - t0)
            t["read_records"].append(t2 - t1)
            t["record_apply_actual"].append(t3 - t2)
            t["apply_records"].append(t4 - t3)
            equal = equal and cs.diff(base) == [] and np.array_equal(rr, rec["rec_at"])
        out = {
            "workload": f"configs[{args.config}] {n} objects, {args.rows} rows + {args.deleted} deleted keys",
            "device": bench._device_info(torch.cuda.current_device()),
            **{k: stats(v) for k, v in t.items()},
            "sizes": {"zones_total": int(snap.actual.n_zones), "records_total": int(snap.actual.n_records), "lbs": int(rs.lb_rows.size),
                      "accels": int(rs.acc_rows.size), "zones": int(rs.zone_rows.size), "zone_records": int(zone_cols["rec_type"].size),
                      "records": int(rr.size), "record_zones": int(rec["zone_target"].size)},
            "delta_bytes": {"zone_apply_actual": delta_bytes(zone_cols), "record_apply_actual": delta_bytes(aws_cols), "apply_records": delta_bytes(rec["rows"])},
            "equal": bool(equal),
        }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
