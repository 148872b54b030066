#!/usr/bin/env python3
"""Cost of `haphic plot` on one GPU host, at the C3 shape (50k contigs, 200M device-resident records from synth) with the
true-layout AGP (synth.write_agp):

  * contact build (count + symmetrise) at 500 kb and 100 kb bins, synchronised host clock, median of --reps;
  * the counting kernel alone on a stream whose every record lands in one bin pair (the worst contention);
  * KR: every scaffold block and the whole matrix balanced together, and the normalised-matrix + median pass;
  * run() wall time from a .pairs file of --file_pairs records (default KR, 500 kb, no figure without matplotlib).

    python scripts/plot_probe.py [--contigs 50000] [--pairs 200000000] [--file_pairs 5000000] [--reps 3] [--out F]

Prints one JSON line (also written to --out) with the card name and power limit."""

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as exc:
        return "unknown ({})".format(exc)


def timed(fn, ctx):
    ctx.sync()
    t = time.perf_counter()
    r = fn()
    ctx.sync()
    return time.perf_counter() - t, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=50_000)
    ap.add_argument("--pairs", type=int, default=200_000_000)
    ap.add_argument("--file_pairs", type=int, default=5_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="plot_probe.json")
    a = ap.parse_args()

    import torch
    from haphic_b200 import plot, synth
    from haphic_b200._lib import Context

    res = {"card": card(), "contigs": a.contigs, "pairs": a.pairs}
    tmp = tempfile.mkdtemp()
    asm = synth.make_assembly(nchr=24, n_contigs=a.contigs, mean_len=3_000_000_000 // a.contigs, seed=31)
    agp = os.path.join(tmp, "c3.agp")
    synth.write_agp(asm, agp)
    rec = synth.make_pairs(asm, a.pairs, seed=32, device="cuda")
    with Context(0) as ctx:
        for kb in (500, 100):
            L = plot.Layout(agp, kb * 1000, 1)
            key = "{}kb".format(kb)
            res[key + "_bins"] = L.nb
            builds, krs, norms = [], [], []
            for _ in range(a.reps + 1):
                cm = plot.ContactMap(ctx, L)
                t, _ = timed(lambda: (cm.add(rec, asynchronous=True), cm.finish()), ctx)
                builds.append(t)
                blocks = L.blocks()
                t, kr = timed(lambda: cm.kr(blocks + [(0, L.nb)]), ctx)
                krs.append(t)
                xb = np.ones(L.nb)
                for (o, n), r in zip(blocks, kr[:-1]):
                    xb[o:o + n] = r[0]
                t, _ = timed(lambda: cm.normalize("KR", blocks, xb, kr[-1][0], want_matrix=True), ctx)
                norms.append(t)
                res[key + "_count_bytes"] = cm.count_bytes
                cm.close()
            res[key + "_build_s"] = float(np.median(builds[1:]))
            res[key + "_records_per_s"] = a.pairs / res[key + "_build_s"]
            res[key + "_kr_s"] = float(np.median(krs[1:]))
            res[key + "_kr_steps_whole"] = list(kr[-1][1:3])
            res[key + "_kr_inner_max_block"] = max(r[2] for r in kr[:-1])
            res[key + "_normalize_s"] = float(np.median(norms[1:]))
            print(json.dumps({k: v for k, v in res.items() if k.startswith(key)}), flush=True)
        # contention: every record in one bin pair (the matrix from the 500 kb layout)
        L = plot.Layout(agp, 500_000, 1)
        hot = rec[:1].repeat(a.pairs // 4, 1).contiguous()
        ts = []
        for _ in range(a.reps + 1):
            cm = plot.ContactMap(ctx, L)
            t, _ = timed(lambda: cm.add(hot, asynchronous=True), ctx)
            ts.append(t)
            cm.close()
        res["one_bin_pair_records_per_s"] = hot.shape[0] / float(np.median(ts[1:]))
        del hot
        # run() from a .pairs file
        sub = rec[:a.file_pairs].cpu().numpy()
        del rec
        torch.cuda.empty_cache()
        pairs = os.path.join(tmp, "aln.pairs")
        synth.write_pairs(asm, sub, pairs)
        res["file_pairs"] = int(sub.shape[0])
        res["file_bytes"] = os.path.getsize(pairs)
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            t0 = time.perf_counter()
            plot.run(plot.parse_arguments([agp, pairs]), ctx=ctx)
            res["run_pairs_file_s"] = time.perf_counter() - t0
        finally:
            os.chdir(cwd)
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
