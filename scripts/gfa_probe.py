#!/usr/bin/env python3
"""Cost of the --gfa phasing at the C3 shape (50k contigs, 200M pairs, two haplotypes) on one GPU:

  * device time of LinkTable.to_matrix, phased (hh_matrix_from_links_phased, w = 1 and w = 0.5) against unphased, timed
    with CUDA events after warm-up, the variants alternating in one process;
  * the contig-level full-link reduction on the device (LinkTable.fetch_phased, reduction and copy to the host) against the
    host reduction of the fetched arrays (LinkArrays.reduce_phasing);
  * one inflation's statistics (output_statistics) on int / float links after w = 0.5, device path (hh_stats) against the
    host path (HAPHIC_STATS_DEVICE=0), and on the integer links; plus the device ranking and best-group kernels alone.

    python scripts/gfa_probe.py [--contigs 50000] [--pairs 200000000] [--reps 5] [--out gfa_probe.json]

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
    except Exception as exc:          # the numbers are still reported, with the failure instead of the card
        return "unknown ({})".format(exc)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=50000)
    ap.add_argument("--pairs", type=int, default=200_000_000)
    ap.add_argument("--nchr", type=int, default=24)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from haphic_b200 import cluster, synth
    ctx = cluster._context()
    dev = torch.device("cuda", ctx.device)
    asm = synth.make_assembly(a.nchr, a.contigs, 20000, seed=2024)
    names = list(asm.names)
    from haphic_b200.links import LinkTable, name_rank
    table = LinkTable(ctx, asm.lengths, name_rank(names), np.ones(asm.n, np.uint8), 500 * 1000,
                      capacity_hint=0)
    step = 1 << 25
    for lo in range(0, a.pairs, step):
        table.add(synth.make_pairs_range(asm, lo, min(a.pairs, lo + step), seed=2025, device=dev), stream_offset=lo)
    table.finish()
    hap = (asm.chrom % 2).astype(np.int32)
    keep = np.ones(asm.n, np.uint8)
    variants = [("unphased", None, 0.0), ("phased_w1", hap, 1.0), ("phased_w0.5", hap, 0.5)]
    times = {v[0]: [] for v in variants}
    nnz = {}
    for rep in range(a.reps + 1):                  # rep 0 is the warm-up of every variant
        for tag, h, w in variants:
            index, n_linked = table.linked_index(keep, hap=h, phasing_weight=w)
            tail = np.nonzero(index < 0)[0].astype(np.int32)
            torch.cuda.synchronize(dev)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            m = table.to_matrix(keep, tail, hap=h, phasing_weight=w)
            end.record()
            torch.cuda.synchronize(dev)
            if rep:
                times[tag].append(start.elapsed_time(end))
            nnz[tag] = m.nnz
            m.close()
    res = dict(card=card(), contigs=a.contigs, pairs=a.pairs, table_nnz=int(table.info.nnz_full))
    for tag in times:
        t = np.array(times[tag])
        res["to_matrix_ms_" + tag] = dict(median=float(np.median(t)), min=float(t.min()), max=float(t.max()), nnz=nnz[tag])

    # full-link reduction: on the device before the fetch, against the host pass over the fetched arrays
    f = table.fetch()
    base = cluster.LinkArrays(names, f["key_i"], f["key_j"], f["full"])
    fa_dict = {n: [None, int(ln), 10] for n, ln in zip(names, asm.lengths.tolist())}
    per = asm.n // a.nchr
    groups = [([names[c] for c in range(g * per, (g + 1) * per)], 0) for g in range(a.nchr)]
    phased = {}
    for w in (1.0, 0.5):
        dev_s = []
        for rep in range(a.reps + 1):
            t0 = time.perf_counter()
            phased[w] = cluster.LinkArrays.from_phased(names, table.fetch_phased(hap, w))
            if rep:
                dev_s.append(time.perf_counter() - t0)
        arr = cluster.LinkArrays(names, f["key_i"], f["key_j"], f["full"])
        t0 = time.perf_counter()
        arr.reduce_phasing(hap, w)
        res["full_link_reduction_s_w{}".format(w)] = dict(device_median=float(np.median(dev_s)), device_min=float(min(dev_s)),
                                                          host=time.perf_counter() - t0)
        res["full_links_after_w{}".format(w)] = len(arr)
        assert len(phased[w]) == len(arr) and np.array_equal(phased[w].values.astype(np.float64), arr.values.astype(np.float64))
    table.close()

    # statistics of one inflation: int / float links on the device and on the host, integer links
    arr = phased[0.5]
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            os.makedirs("inflation_1", exist_ok=True)
            for tag, links, env in (("int", base, "1"), ("float_device", arr, "1"), ("float_host", arr, "0")):
                os.environ["HAPHIC_STATS_DEVICE"] = env
                reps = 1 if tag == "float_host" else a.reps
                t = []
                for rep in range(reps + 1):
                    t0 = time.perf_counter()
                    cluster.output_statistics(fa_dict, links, [(1, groups)])
                    if rep:
                        t.append(time.perf_counter() - t0)
                res["statistics_s_" + tag] = float(np.median(t))
        finally:
            os.chdir(cwd)
            os.environ.pop("HAPHIC_STATS_DEVICE", None)
    # the device kernels of one inflation alone (rank + best-group statistics, CUDA events on the library's stream)
    st = arr.stats_device(ctx)
    gid = np.repeat(np.arange(a.nchr, dtype=np.int32), per)
    gid = np.concatenate([gid, np.full(asm.n - len(gid), -1, np.int32)])
    gre, cre = np.full(a.nchr, 1 + 9 * per, np.int64), np.full(asm.n, 10, np.int64)
    ms = []
    for rep in range(a.reps + 1):
        stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(stream)
        nseg = st.rank(gid, a.nchr)
        st.best(gre, cre, compensated=True)
        end.record(stream)
        end.synchronize()
        if rep:
            ms.append(start.elapsed_time(end))
    res["stats_device_ms"] = dict(median=float(np.median(ms)), min=float(min(ms)), max=float(max(ms)), segments=int(nseg),
                                  directed_entries=2 * len(arr))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fo:
            fo.write(line + "\n")


if __name__ == "__main__":
    main()
