"""Matrix-stage probe at C3 (50k contigs / 200M pairs): device time of linked_index + to_matrix, the way bench.py calls
them, each time on a newly built link table (so the index is computed, not reused).

    python scripts/matrix_probe.py                      # event-timed warm repetitions (REPS, default 10), each on a new table
    python scripts/matrix_probe.py --profile OUT_DIR    # per-kernel device times of one stage (torch.profiler)

The profile mode runs one warm-up stage, then profiles linked_index and to_matrix in two separate profiler sessions and
writes OUT_DIR/matrix_kernels.json (total and per-launch device time of every kernel and copy, per call) and a Chrome
trace of each.  Both modes report this process's device memory (NVML) after the table build and after the matrix: the
library keeps freed blocks in its pools, so the second figure is the process's high-water mark over build + matrix.
Where NVML does not list the process (a PID namespace), the figure is the growth of the whole device's used memory
since start-up instead, and says so."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from haphic_b200 import synth
from haphic_b200._lib import Context
from haphic_b200.links import LinkTable, name_rank

ap = argparse.ArgumentParser()
ap.add_argument("--profile", metavar="OUT_DIR", help="per-kernel device times of the matrix stage under OUT_DIR")
args = ap.parse_args()

def _device_used():
    free, total = torch.cuda.mem_get_info(0)
    return total - free


_base = _device_used()                     # before the records, the context and the table


pairs = int(os.environ.get("PAIRS", "200000000"))
asm = synth.make_assembly(24, 50000, 20000, seed=12345)
rank = name_rank(asm.names)
in_nx = np.ones(asm.n, np.uint8)
rec = synth.make_pairs_range(asm, 0, pairs, seed=12346, device="cuda")
ctx = Context(0)
stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
keep = np.ones(asm.n, np.uint8)


def used_gb():
    """(GB, source) of this process's device memory"""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        for p in pynvml.nvmlDeviceGetComputeRunningProcesses(h):
            if p.pid == os.getpid() and p.usedGpuMemory:
                return round(p.usedGpuMemory / 1e9, 2), "nvml process"
    except Exception:
        pass
    return round((_device_used() - _base) / 1e9, 2), "device growth since start-up"


def build():
    tab = LinkTable(ctx, asm.lengths, rank, in_nx, 500000, capacity_hint=int(0.45 * pairs))
    tab.add(rec, asynchronous=True)
    info = tab.finish()
    ctx.sync()
    return tab, info


tab, info = build()
mem_build = used_gb()


def stage(tab, ev=None):
    """linked_index + to_matrix as bench.py runs them, on a table that has computed no index yet"""
    if ev:
        ev[0].record(stream)
    index, _ = tab.linked_index(keep)
    if ev:
        ev[1].record(stream)
    mat = tab.to_matrix(keep, np.nonzero(index < 0)[0].astype(np.int32))
    if ev:
        ev[2].record(stream)
        ev[2].synchronize()
    mat.close()


head = {"gpu": torch.cuda.get_device_name(0), "pairs": pairs, "nnz_full": int(info.nnz_full), "nnz_flank": int(info.nnz_flank)}

if args.profile:
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(args.profile, exist_ok=True)
    stage(tab)
    tab.close()
    tab, _ = build()
    calls = {}
    for call in ("linked_index", "to_matrix"):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            if call == "linked_index":
                index, _ = tab.linked_index(keep)
                ctx.sync()
            else:
                mat = tab.to_matrix(keep, np.nonzero(index < 0)[0].astype(np.int32))
                ctx.sync()
        kernels = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                name = e.name.split("(")[0].replace("void ", "")
                k = kernels.setdefault(name, {"launches": 0, "ms": 0.0})
                k["launches"] += 1
                k["ms"] += e.time_range.elapsed_us() / 1000.0
        for k in kernels.values():
            k["ms_per_launch"] = k["ms"] / k["launches"]
        calls[call] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms"]))
        prof.export_chrome_trace(os.path.join(args.profile, "matrix_trace_{}.json".format(call)))
    mem_matrix = used_gb()
    mat.close()
    out = dict(head, mem_gb_after_build=mem_build, mem_gb_after_matrix=mem_matrix, kernels=calls)
    with open(os.path.join(args.profile, "matrix_kernels.json"), "w") as f:
        json.dump(out, f, indent=1)
    for call, kernels in calls.items():
        print(call)
        for name, k in kernels.items():
            print("{:>9.3f} ms  {:>5d} x  {}".format(k["ms"], k["launches"], name[:110]))
    print("device memory of the process: {} after build, {} after matrix".format(mem_build, mem_matrix))
    sys.exit(0)

stage(tab)
t_index, t_matrix = [], []
for rep in range(int(os.environ.get("REPS", "10"))):
    tab.close()
    tab, _ = build()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    stage(tab, ev)
    t_index.append(ev[0].elapsed_time(ev[1]))
    t_matrix.append(ev[1].elapsed_time(ev[2]))
tot = [a + b for a, b in zip(t_index, t_matrix)]
print(json.dumps(dict(head, mem_gb_after_build=mem_build, mem_gb_after_matrix=used_gb(),
                      linked_index_ms=[round(x, 3) for x in t_index], to_matrix_ms=[round(x, 3) for x in t_matrix],
                      stage_ms_median=round(float(np.median(tot)), 3), stage_ms_min=round(min(tot), 3),
                      stage_ms_max=round(max(tot), 3))))
tab.close()
