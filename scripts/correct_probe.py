"""Assembly-correction probe at the C3 shape (50k contigs, 200M pairs) with planted chimeras: device time of every phase
of `--correct_nrounds 2` (coverage pass, the two rounds, remap) next to the link build of the remapped stream, the
intra-contig fraction of the stream, and the card it ran on.  Device times are for device-resident records;
host_path_ms gives the wall times of the path cluster.run() takes (host record batches, copies both ways).  Prints one
JSON line.  PAIRS / JOINS override the shape."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from haphic_b200 import synth
from haphic_b200._lib import Context
from haphic_b200.correct import Correction
from haphic_b200.links import LinkTable, name_rank

pairs = int(os.environ.get("PAIRS", "200000000"))
n_joins = int(os.environ.get("JOINS", "500"))
res = 500
dev = torch.device("cuda", 0)
asm = synth.make_assembly(24, 50000, 20000, seed=12345)
rec = synth.make_pairs_range(asm, 0, pairs, seed=12346, device=dev)
# chimeras: contig a + contig b of another chromosome, as synth.make_chimeras lays them out, mapped on the device
rng = np.random.default_rng(7)
per_chr = asm.n // 24
picks = rng.permutation(per_chr)[:2 * n_joins]
joins = [(int(picks[2 * k]), int(picks[2 * k + 1]) + per_chr * (1 + k % 23)) for k in range(n_joins)]
joined = {c for j in joins for c in j}
keep = [c for c in range(asm.n) if c not in joined]
new_id = np.full(asm.n, -1, np.int64)
off = np.zeros(asm.n, np.int64)
new_id[keep] = np.arange(len(keep))
lengths = [int(asm.lengths[c]) for c in keep]
for k, (a, b) in enumerate(joins):
    new_id[a] = new_id[b] = len(lengths)
    off[b] = asm.lengths[a]
    lengths.append(int(asm.lengths[a] + asm.lengths[b]))
nid, noff = torch.from_numpy(new_id).to(dev), torch.from_numpy(off).to(dev)
for s in (0, 2):
    c = rec[:, s].long()
    rec[:, s + 1] += noff[c].to(torch.int32)
    rec[:, s] = nid[c].to(torch.int32)
lengths = np.asarray(lengths, np.int64)
n = len(lengths)
intra = float((rec[:, 0] == rec[:, 2]).float().mean())

ctx = Context(0)
stream = torch.cuda.ExternalStream(ctx.stream)


def timed(fn):
    ctx.sync()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    out = fn()
    b.record(stream)
    b.synchronize()
    return out, a.elapsed_time(b)


result = {}
for rep in range(int(os.environ.get("REPS", "3"))):
    corr = Correction(ctx, lengths, res)
    _, t_cov = timed(lambda: corr.add(rec))
    i1, t_r1 = timed(lambda: corr.round(0.2, 0.1, 5000, False))
    i2, t_r2 = timed(lambda: corr.round(0.2, 0.1, 5000, True))
    # the remap's cost does not depend on the names the host gives the pieces: every contig keeps its id here
    corr.set_layout(np.arange(n + 1), np.zeros(n, np.int64), np.arange(n))
    out, t_remap = timed(lambda: corr.remap(rec))
    corr.close()
    tab = LinkTable(ctx, lengths, name_rank(["c{}".format(i) for i in range(n)]), np.ones(n, np.uint8), 500000,
                    capacity_hint=int(0.45 * pairs))
    _, t_links = timed(lambda: (tab.add(out, asynchronous=True), tab.finish()))
    tab.close()
    del out
    result = dict(records=pairs, contigs=n, planted_chimeras=n_joins, intra_fraction=round(intra, 4),
                  n_links=int(i1.n_links), broken_round1=int(i1.n_broken), broken_round2=int(i2.n_broken),
                  coverage_ms=round(t_cov, 2), round1_ms=round(t_r1, 2), round2_ms=round(t_r2, 2), remap_ms=round(t_remap, 2),
                  link_build_ms=round(t_links, 2),
                  correction_over_link_build=round((t_cov + t_r1 + t_r2 + t_remap) / t_links, 3), rep=rep)
    print(json.dumps(result), file=sys.stderr, flush=True)
# the path cluster.run() takes: host record batches as the readers yield them (4M records), copied to the device for the
# coverage pass and for the remap, remapped batches back on the host (CLM writer) and copied again by the link build
host = rec.cpu().numpy()
del rec
batches = [host[k:k + 4_000_000] for k in range(0, len(host), 4_000_000)]
ctx.sync()
t0 = time.perf_counter()
corr = Correction(ctx, lengths, res)
for b in batches:
    corr.add(b)
t1 = time.perf_counter()
corr.round(0.2, 0.1, 5000, False)
corr.round(0.2, 0.1, 5000, True)
corr.set_layout(np.arange(n + 1), np.zeros(n, np.int64), np.arange(n))
t2 = time.perf_counter()
remapped = [corr.remap(b, in_place=True) for b in batches]
t3 = time.perf_counter()
corr.close()
tab = LinkTable(ctx, lengths, name_rank(["c{}".format(i) for i in range(n)]), np.ones(n, np.uint8), 500000)
for b in remapped:
    tab.add(b)
tab.finish()
ctx.sync()
t4 = time.perf_counter()
tab.close()
result["host_path_ms"] = dict(coverage=round(1e3 * (t1 - t0), 1), rounds=round(1e3 * (t2 - t1), 1), remap=round(1e3 * (t3 - t2), 1),
                              link_build=round(1e3 * (t4 - t3), 1), host_bytes_kept=int(host.nbytes))
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
result["gpu"] = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else torch.cuda.get_device_name(0)
print(json.dumps(result))
