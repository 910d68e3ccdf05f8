"""Slab compaction against the reload it replaces: one JSON line on stdout.

  python profiles/compact_bench.py [--config 3] [--objects 1000000] [--churn 0.1] [--max-batches 12] [--reps 5] [--seed 17]

Workload: bench.py's timed snapshot (BASELINE configs[2] at 10^6 objects, column-major slabs, rank 0's seed).  Batches of
deltas.churn and deltas.aws_churn (deterministic from --seed) are applied to the table-level mirrors until both slabs have grown
by at least 50 % (or --max-batches is reached; the growth reached is reported).  The mirrors then hold the tables of a delta-fed
engine byte for byte ("grown"), and their compact() the tables a compaction leaves ("compacted").  Reported, medians over --reps
repetitions with min / max:
  compact   gar_snapshot_compact of one group on a freshly loaded grown snapshot: host clock around the call, which ends in a
            device synchronise (allocation of the new slab and release of the old one included).  bytes = what the algorithm
            must move, from the tables: every live string byte read and written once (2 x live) plus 80 bytes per string for
            its references and offsets (lengths pass 8 + 16, scan 16, copy 16, rewrite 16 + 8); GB/s = bytes / time, and its
            share of 3.35 TB/s, the H100 SXM data-sheet HBM bandwidth (a denominator, not a measured peak);
  load      gar_snapshot_load of the compacted tables from pinned host memory: the reload a worker would do instead;
  diff      the full diff with GAR_FLAG_REPREPARE (device time, ms_kernels) on three engines, alternating: the grown snapshot,
            the same after gar_snapshot_compact of both groups, and a fresh load of the compacted tables;
  equal     the three change sets agree: tok_name / tok_region as the strings they name, every other array bit for bit.
Like bench.py it runs on the tree as __graft_entry__.build() left it and writes nothing into it.
"""
import argparse
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

HBM_DATASHEET = 3.35e12
REF_BYTES_PER_STRING = 80
OBJ, ACT = 1, 2


def stats(v):
    return {"median": round(float(np.median(v)), 3), "min": round(float(min(v)), 3), "max": round(float(max(v)), 3)}


def n_strings(cols, tables_def):
    return int(sum(len(cols[name]) for _, (_, cl) in tables_def.items() for name, kind in cl if kind == "str" and name != "obj_name"))


def tok_strings(refs, slab):
    off = (refs & np.uint64((1 << 40) - 1)).astype(np.int64)
    ln = (refs >> np.uint64(40)).astype(np.int64)
    idx = np.repeat(off - np.concatenate([[0], np.cumsum(ln)[:-1]]), ln) + np.arange(int(ln.sum()), dtype=np.int64)
    return ln, slab[idx]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--objects", type=int, default=1_000_000)
    ap.add_argument("--churn", type=float, default=0.1)
    ap.add_argument("--max-batches", type=int, default=12)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=17)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("compact_bench.py needs a CUDA device: the engine has no CPU path")
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
    batches = 0
    while batches < args.max_batches and (om.slab_len < 1.5 * loaded[0] or am.slab_len < 1.5 * loaded[1]):
        up, deleted = deltas.churn(om, rng, frac=args.churn, serial=batches)
        keep, uobj = deltas.objects_struct(up)
        res = eng.apply_objects(uobj, deleted)
        om.apply(up, deleted)
        d = deltas.aws_churn(am, rng, frac=args.churn, max_zones=zones)
        keep2, rows = deltas.actual_struct(d["rows"])
        ares = eng.apply_actual(rows, d["lb_target"], d["acc_target"], d["zone_target"], d["lb_deleted"], d["acc_deleted"])
        am.apply(**d)
        if (res.slab_len, ares.slab_len) != (om.slab_len, am.slab_len):
            raise RuntimeError("the engine's slab lengths differ from the table-level mirrors'")
        batches += 1
    grown = tables.from_columns(om.cur, am.cur)
    grown_len = (om.slab_len, am.slab_len)
    strings = (n_strings(om.cur, tables.OBJ_TABLES), n_strings(am.cur, tables.ACT_TABLES))

    # (a) the delta-fed engine first (its slabs grew by reallocation), then freshly loaded grown snapshots
    ms = {OBJ: [], ACT: []}
    live = None
    for rep in range(args.reps + 1):
        if rep:
            eng.load(grown)
        for g in (OBJ, ACT):
            t0 = time.perf_counter()
            r = eng.compact(g)
            ms[g].append((time.perf_counter() - t0) * 1e3)
        live = (int(r.obj_slab_len), int(r.act_slab_len))
    first = {"objects": round(ms[OBJ][0], 3), "actual": round(ms[ACT][0], 3)}
    if live != (om.compact(), am.compact()):
        raise RuntimeError("the compacted slab lengths differ from the table-level mirrors'")
    compacted = tables.from_columns(om.cur, am.cur)

    def rate(g, k):
        t = float(np.median(ms[g][1:])) * 1e-3
        nbytes = 2 * live[k] + REF_BYTES_PER_STRING * strings[k]
        return {"ms": stats(ms[g][1:]), "live_slab_bytes": live[k], "strings": strings[k], "bytes_moved": nbytes, "GBps": round(nbytes / t / 1e9, 1),
                "share_of_datasheet_3.35TBps": round(nbytes / t / HBM_DATASHEET, 4)}

    out = {"device": bench._device_info(torch.cuda.current_device()),
           "config": {"workload": f"BASELINE configs index {args.config}, {args.objects} objects, column-major slabs", "seed": int(cfg.seed),
                      "churn": args.churn, "churn_seed": args.seed, "batches": batches, "zones_per_batch": zones, "reps": args.reps},
           "slab_growth": {"objects": round(grown_len[0] / loaded[0], 3), "actual": round(grown_len[1] / loaded[1], 3)},
           "compact_objects": rate(OBJ, 0), "compact_actual": rate(ACT, 1), "ms_first_compact_of_delta_fed_engine": first}

    # (b) the reload it replaces
    _, pins = bench._pin_host_tables(torch, abi, compacted.objects, compacted.actual)
    loads = []
    for _ in range(args.reps + 1):
        t0 = time.perf_counter()
        eng.load(compacted)
        loads.append((time.perf_counter() - t0) * 1e3)
    bench._unpin(torch, pins)
    out["ms_load_compacted_pinned"] = stats(loads[1:])
    out["load_h2d_bytes"] = int(sum(int(c) * s for (_, c, s) in bench._table_arrays(abi, compacted.objects, compacted.actual)))
    eng.close()

    # (c) the full diff on the three layouts, alternating
    arms = {"grown": pkg.Engine(cluster_name=snap.cluster, reprepare=True), "compacted_on_device": pkg.Engine(cluster_name=snap.cluster, reprepare=True),
            "fresh_load_of_compacted": pkg.Engine(cluster_name=snap.cluster, reprepare=True)}
    arms["grown"].load(grown)
    arms["compacted_on_device"].load(grown)
    arms["compacted_on_device"].compact(OBJ | ACT)
    arms["fresh_load_of_compacted"].load(compacted)
    diff_ms = {k: [] for k in arms}
    for rep in range(2 * args.reps + 2):
        for k, e in arms.items():
            t = e.diff_device().ms_kernels
            if rep >= 2:
                diff_ms[k].append(t)
    out["ms_full_diff_reprepare"] = {k: stats(v) for k, v in diff_ms.items()}

    # (d) the three change sets agree
    slabs = {"grown": np.asarray(om_slab(grown)), "compacted_on_device": arms["compacted_on_device"].read_slab(OBJ, 0, live[0]),
             "fresh_load_of_compacted": np.asarray(om_slab(compacted))}
    sets = {k: e.diff() for k, e in arms.items()}
    ref, bad = sets["grown"], []
    for k in ("compacted_on_device", "fresh_load_of_compacted"):
        for name in ref.ARRAYS:
            a, b = getattr(ref, name), getattr(sets[k], name)
            if name in ("tok_name", "tok_region"):
                (la, sa), (lb, sb) = tok_strings(a, slabs["grown"]), tok_strings(b, slabs[k])
                same = np.array_equal(la, lb) and np.array_equal(sa, sb)
            else:
                same = a.shape == b.shape and np.array_equal(a, b)
            if not same:
                bad.append(f"{k}.{name}")
    out["equal"] = not bad
    if bad:
        out["mismatch"] = bad
    for e in arms.values():
        e.close()
    print(json.dumps(out), flush=True)


def om_slab(snap):
    return snap.arrays["o.slab"][:int(snap.objects.slab_len)]


if __name__ == "__main__":
    main()
