#!/usr/bin/env python3
"""Cost of `haphic cluster --ul` on one GPU host:

  * the native UL reader (hh_ul_open: threaded BGZF inflate, then the record walk and the primary / supplementary state
    machine on one thread) on a synthetic UL BAM of at least --gb GB: reads across the junctions of consecutive contigs
    (synth.ul_reads) with random SEQ / QUAL, the compressed records repeated until the file is large enough; wall time of
    ul.read_ul_events per call, file bytes / s and records / s, median of --reads calls (the first call reads the file
    from disk, later ones from the page cache: both are reported);
  * C3 shape (50k contigs, 200M pairs): LinkTable.to_matrix without and with the UL arrays (about 2,000 paths of five
    consecutive contigs), CUDA events around the call after warm-up, the two variants alternating, medians of --reps.

    python scripts/ul_probe.py [--gb 5] [--reads 3] [--contigs 50000] [--pairs 200000000] [--reps 5] [--tmp DIR] [--out F]

The BAM goes to a temporary directory (under --tmp) that is removed at the end.  Prints one JSON line (also written to
--out) with the card name and power limit."""

import argparse
import json
import os
import shutil
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


def reader(a, res):
    from argparse import Namespace
    from haphic_b200 import hicio, synth, ul
    asm = synth.make_assembly(24, 2400, 100000, seed=3100)
    names, lengths, recs = synth.ul_reads(asm, 3101, support=3, keep=0.9)
    tmp = tempfile.mkdtemp(prefix="ul_probe_", dir=a.tmp)
    try:
        path = os.path.join(tmp, "ul.bam")
        # one copy of the records, to learn its compressed size, then as many copies as reach --gb
        hicio.write_ul_bam(path, names, lengths, recs, random_seq=np.random.default_rng(3102))
        one = os.path.getsize(path)
        repeat = max(1, int(np.ceil(a.gb * 1e9 / one)))
        t0 = time.perf_counter()
        hicio.write_ul_bam(path, names, lengths, recs, repeat=repeat, random_seq=np.random.default_rng(3102))
        size = os.path.getsize(path)
        args = Namespace(threads=a.threads, min_ul_mapq=30, min_ul_alignment_length=10000, max_distance_to_end=100,
                         max_overlap_ratio=0.5, max_gap_len=10000)
        secs, n_events = [], 0
        for _ in range(a.reads):
            t = time.perf_counter()
            _n, _l, ev = ul.read_ul_events(path, args)
            secs.append(time.perf_counter() - t)
            n_events = len(ev)
        n_rec = len(recs) * repeat
        res["ul_reader"] = dict(file_bytes=size, records=n_rec, events=n_events, threads=a.threads, write_s=time.perf_counter() - t0,
                                seconds=secs, first_s=secs[0], median_s=float(np.median(secs)),
                                median_gb_per_s=size / float(np.median(secs)) / 1e9,
                                median_records_per_s=n_rec / float(np.median(secs)))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def matrix(a, res):
    import torch
    from haphic_b200 import cluster, synth
    from haphic_b200.links import LinkTable, name_rank
    ctx = cluster._context()
    dev = torch.device("cuda", ctx.device)
    asm = synth.make_assembly(24, a.contigs, 20000, seed=2024)
    names = list(asm.names)
    table = LinkTable(ctx, asm.lengths, name_rank(names), np.ones(asm.n, np.uint8), 500 * 1000, capacity_hint=0)
    step = 1 << 25
    for lo in range(0, a.pairs, step):
        table.add(synth.make_pairs_range(asm, lo, min(a.pairs, lo + step), seed=2025, device=dev), stream_offset=lo)
    table.finish()
    n = asm.n
    rng = np.random.default_rng(3103)
    path = np.full(n, -1, np.int32)
    for k, blk in enumerate(rng.choice(n // 5, min(2000, n // 5), replace=False).tolist()):
        path[5 * blk:5 * blk + 5] = k
    ul_arrays = (path, np.arange(n, dtype=np.int32))
    keep = np.ones(n, np.uint8)
    index, _n_linked = table.linked_index(keep)
    tail = np.nonzero(index < 0)[0].astype(np.int32)
    variants = [("plain", None), ("ul", ul_arrays)]
    times = {v[0]: [] for v in variants}
    nnz = {}
    for rep in range(a.reps + 1):                  # rep 0 is the warm-up of both variants
        for tag, u in variants:
            torch.cuda.synchronize(dev)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            m = table.to_matrix(keep, tail, ul=u)
            end.record()
            torch.cuda.synchronize(dev)
            if rep:
                times[tag].append(start.elapsed_time(end))
            nnz[tag] = m.nnz
            m.close()
    table.close()
    res["contigs"], res["pairs"] = a.contigs, a.pairs
    for tag, t in times.items():
        t = np.array(t)
        res["to_matrix_ms_" + tag] = dict(median=float(np.median(t)), min=float(t.min()), max=float(t.max()), nnz=nnz[tag])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=5.0)
    ap.add_argument("--reads", type=int, default=3)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--contigs", type=int, default=50000)
    ap.add_argument("--pairs", type=int, default=200_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--tmp", default=None)
    ap.add_argument("--skip_reader", action="store_true")
    ap.add_argument("--skip_matrix", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    if not a.skip_reader:
        reader(a, res)
    if not a.skip_matrix:
        matrix(a, res)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
