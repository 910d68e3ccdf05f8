"""gar_read_set on a prepared snapshot, and the refresh loop it enables: one JSON line on stdout.

  python profiles/read_set_bench.py [--config 2] [--objects 1000000] [--rows 10000] [--deleted 100] [--reps 11] [--seed 17]

Workload: bench.py's timed snapshot (BASELINE configs[2] at 10^6 objects, column-major slabs, rank 0's seed).  The keyset is
--rows object rows drawn with --seed plus the keys of --deleted other objects passed as deleted keys (their cleanup walks
ix_owner / ix_val).  Reported, medians over --reps with min and max, host clock around calls that synchronise:
  read_set      gar_read_set of the keyset on a prepared snapshot, and the sizes of the set;
  diff_keys     gar_diff_keys of the keyset on a prepared snapshot (today's loop);
  loop          gar_read_set -> gar_snapshot_apply_actual of those rows re-described unchanged -> gar_diff_keys (the first diff
                after an AWS delta re-prepares the snapshot).
`equal`: the loop's change set equals the plain gar_diff_keys'.  Like bench.py it runs on the tree as __graft_entry__.build()
left it and writes nothing into it.
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


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


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
        raise SystemExit("read_set_bench.py needs a CUDA device: the engine has no CPU path")
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
        e.diff_keys(rows, deleted)  # prepares the snapshot and builds ix_owner / ix_val
        e.read_set(rows, deleted)
        t_rs, t_dk, t_loop = [], [], []
        for _ in range(args.reps):
            t, rs = timed(lambda: e.read_set(rows, deleted))
            t_rs.append(t)
            t, base = timed(lambda: e.diff_keys(rows, deleted))
            t_dk.append(t)
        # the loop, with the rows re-described unchanged (taken from the loaded tables, outside the timed window: a worker gets
        # them from AWS): the resident tables stay what they were
        equal = True
        for _ in range(args.reps):
            rs = e.read_set(rows, deleted)
            keep, delta = deltas.actual_struct(deltas.compact_actual(deltas.actual_rows(act, rs.lb_rows, rs.acc_rows, rs.zone_rows)))
            t0 = time.perf_counter()
            rs = e.read_set(rows, deleted)
            e.apply_actual(delta, rs.lb_rows, rs.acc_rows, rs.zone_rows)
            cs = e.diff_keys(rows, deleted)
            t_loop.append(time.perf_counter() - t0)
            equal = equal and cs.diff(base) == []
            del keep
        out = {
            "workload": f"configs[{args.config}] {n} objects, {args.rows} rows + {args.deleted} deleted keys",
            "device": bench._device_info(torch.cuda.current_device()),
            "read_set": stats(t_rs), "diff_keys": stats(t_dk), "loop": stats(t_loop),
            "sizes": {"lbs": int(rs.lb_rows.size), "lb_misses": int(rs.lb_miss_obj.size), "accels": int(rs.acc_rows.size), "zones": int(rs.zone_rows.size)},
            "equal": bool(equal),
        }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
