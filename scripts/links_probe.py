"""Link-counting probe at C3 (50k contigs / 200M pairs): wall / device time of add and finish for the direct and the
partitioned engines.

    python scripts/links_probe.py                      # wall times, MODES (default "0,1") x REPS (default 3)
    python scripts/links_probe.py --profile OUT_DIR    # per-kernel device times of the partitioned engine (torch.profiler)

The profile mode runs one warm-up and one profiled pass of the partitioned engine and writes OUT_DIR/links_kernels.json
(total and per-launch device time of every kernel: scatter, hist, scatter2, bucket count, fallback) and a Chrome trace."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from haphic_b200 import synth
from haphic_b200._lib import Context
from haphic_b200.links import LinkTable, name_rank

ap = argparse.ArgumentParser()
ap.add_argument("--profile", metavar="OUT_DIR", help="per-kernel device times of the partitioned engine under OUT_DIR")
args = ap.parse_args()

pairs = int(os.environ.get("PAIRS", "200000000"))
asm = synth.make_assembly(24, 50000, 20000, seed=12345)
rank = name_rank(asm.names)
in_nx = np.ones(asm.n, np.uint8)
rec = synth.make_pairs_range(asm, 0, pairs, seed=12346, device="cuda")
ctx = Context(0)


def build():
    tab = LinkTable(ctx, asm.lengths, rank, in_nx, 500000, capacity_hint=int(0.45 * pairs))
    tab.add(rec, asynchronous=True)
    info = tab.finish()
    ctx.sync()
    return tab, info


if args.profile:
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(args.profile, exist_ok=True)
    os.environ["HH_LINKS_PARTITION"] = "1"
    os.environ.pop("HH_LINKS_NPART_LOG", None)
    build()[0].close()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        tab, info = build()
    agg = tab.agg_info()
    tab.close()
    kernels = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and e.name.startswith(("hh_k_", "void hh_k_", "_Z")):
            k = kernels.setdefault(e.name, {"launches": 0, "ms": 0.0})
            k["launches"] += 1
            k["ms"] += e.time_range.elapsed_us() / 1000.0
    for k in kernels.values():
        k["ms_per_launch"] = k["ms"] / k["launches"]
    out = {"gpu": torch.cuda.get_device_name(0), "pairs": pairs, "n_used": int(info.n_used), "nnz_full": int(info.nnz_full),
           "agg": agg, "kernels": dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms"]))}
    with open(os.path.join(args.profile, "links_kernels.json"), "w") as f:
        json.dump(out, f, indent=1)
    prof.export_chrome_trace(os.path.join(args.profile, "links_trace.json"))
    for name, k in out["kernels"].items():
        print("{:>9.3f} ms  {:>5d} x  {}".format(k["ms"], k["launches"], name[:110]))
    print("agg", agg)
    sys.exit(0)

for mode in os.environ.get("MODES", "0,1").split(","):
    os.environ["HH_LINKS_PARTITION"] = mode
    for rep in range(int(os.environ.get("REPS", "3"))):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tab = LinkTable(ctx, asm.lengths, rank, in_nx, 500000, capacity_hint=int(0.45 * pairs))
        tab.add(rec, asynchronous=True)
        ctx.sync()
        t1 = time.perf_counter()
        info = tab.finish()
        ctx.sync()
        t2 = time.perf_counter()
        keep = np.ones(asm.n, np.uint8)
        index, _ = tab.linked_index(keep)
        mat = tab.to_matrix(keep, np.nonzero(index < 0)[0].astype(np.int32))
        ctx.sync()
        t3 = time.perf_counter()
        print("mode", mode, "rep", rep, "add ms", round(1e3 * (t1 - t0), 2), "finish ms", round(1e3 * (t2 - t1), 2), "index+matrix ms",
              round(1e3 * (t3 - t2), 2), "nnz", info.nnz_full, "slots", info.table_slots, "agg", tab.agg_info(), flush=True)
        mat.close()
        tab.close()
