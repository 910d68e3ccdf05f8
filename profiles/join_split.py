"""Where the owner-keyed joins and the index builds spend their time, launch by launch: one JSON line on stdout.

  python profiles/join_split.py [--config 3] [--objects 1000000] [--diffs 5]

Runs run_once.py's workload (BASELINE configs[2] at 10^6 objects, column-major slabs, GAR_FLAG_REPREPARE: every diff
prepares the snapshot again) under torch.profiler with CUDA activities, one profiler session per diff, and reports the mean
device time of every kernel of the join stages, told apart by the functor types in the kernel's template name and, where two
launches share one type, by their order inside the diff:
  value_joins       the fused value / accelerator pass of the full prepare (alias link + object resolution)
  resolve_owners    the same pass without the alias link: measured on a second engine without REPREPARE whose object
                    table took one delta (gar_snapshot_apply_objects), so its next full diff re-resolves the owners only
  idx_place.*       group A's placement and the second placement (orphan-value index and owned lists)
  idx_order.*       the ordering launches, in diff order
Kernel names are the template names the profiler shows; a kernel that matches none of the rows is summed under `other`.
Times under the profiler are not bench values.  Needs a CUDA device: the engine has no CPU path.
"""
import argparse
import importlib
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402


def label(name, seen):
    """row of the report for a kernel name; `seen` counts same-named launches inside one diff"""
    if "FValueJoins" in name:
        return "value_joins"
    if "FResolveValue" in name:
        return "resolve_owners"
    if "FIdxPlaceDirect<FRowLb>" in name or "FIdxPlaceDirect<FRowThost>" in name:
        return "idx_place.group_a"
    if "FIdxPlaceDirect<FRowOvn>" in name:
        return "idx_place.ovn_own"
    if "FIdxOrderMulti" in name:
        seen["idx_order"] = seen.get("idx_order", 0) + 1
        return f"idx_order#{seen['idx_order']}"
    return None


def profile_diffs(torch, eng, n):
    from torch.profiler import ProfilerActivity, profile
    per = []
    for _ in range(n):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.diff_device()
            torch.cuda.synchronize()
        ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
        row, seen = {}, {}
        for e in ev:
            k = label(e.name, seen) or "other"
            row[k] = row.get(k, 0.0) + e.device_time / 1e3
            if k != "other":
                row.setdefault("_names", {})[k] = e.name[:160]
        per.append(row)
    keys = sorted({k for r in per for k in r if k != "_names"})
    out = {k: round(float(np.mean([r.get(k, 0.0) for r in per])), 4) for k in keys}
    names = {}
    for r in per:
        names.update(r.get("_names", {}))
    return out, names


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--objects", type=int, default=1_000_000)
    ap.add_argument("--diffs", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("join_split.py needs a CUDA device: the engine has no CPU path")
    import bench
    bench._require_built()
    pkg = importlib.import_module("aws-global-accelerator-controller_b200")
    synth = importlib.import_module("aws-global-accelerator-controller_b200.synth")
    deltas = importlib.import_module("aws-global-accelerator-controller_b200.deltas")
    tables = pkg.tables
    cfg = synth.preset(args.config, args.objects)
    cfg.layout = 1
    snap = synth.SynthSnapshot(cfg)

    with pkg.Engine(cluster_name=snap.cluster, reprepare=True) as e:
        e.load(snap)
        for _ in range(2):
            e.diff_device()
        full, names = profile_diffs(torch, e, args.diffs)

    # resolve_owners(false): one object delta, then the next full diff rebuilds the object side and re-resolves the owners
    mirror = deltas.ColumnMirror(tables.columns(snap.objects, tables.OBJ_TABLES))
    rng = np.random.default_rng(11)
    reres = []
    with pkg.Engine(cluster_name=snap.cluster) as e:
        e.load(snap)
        e.diff_device()
        for b in range(args.diffs + 1):
            up, deleted = deltas.churn(mirror, rng, frac=0.001, serial=b)
            _, uobj = deltas.objects_struct(up)
            e.apply_objects(uobj, deleted)
            mirror.apply(up, deleted)
            r, n2 = profile_diffs(torch, e, 1)
            names.update(n2)
            if b:
                reres.append(r)
    after = {k: round(float(np.mean([r.get(k, 0.0) for r in reres])), 4) for k in sorted({k for r in reres for k in r})}

    join = ("value_joins", "idx_place", "idx_order")
    out = {"device": bench._device_info(torch.cuda.current_device()),
           "config": {"workload": f"BASELINE configs index {args.config}, {args.objects} objects, column-major slabs, REPREPARE",
                      "seed": int(cfg.seed), "diffs": args.diffs},
           "full_diff_ms": full,
           "join_stages_ms": round(sum(v for k, v in full.items() if k.startswith(join)), 4),
           "after_object_delta_ms": after,
           "kernel_names": names}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
