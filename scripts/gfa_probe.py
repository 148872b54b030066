#!/usr/bin/env python3
"""Cost of the --gfa phasing and of the reassignment statistics on one GPU:

  * C3 shape (50k contigs, 200M pairs, two haplotypes): device time of LinkTable.to_matrix, phased
    (hh_matrix_from_links_phased, w = 1 and w = 0.5) against unphased, timed with CUDA events after warm-up, the variants
    alternating in one process;
  * the contig-level full-link reduction on the device (LinkTable.fetch_phased, reduction and copy to the host) against the
    host reduction of the fetched arrays (tests/stats_oracle.py);
  * one inflation's statistics (output_statistics) on the integer links and on the int / float links after w = 0.5 (C3
    shape), and on the reference's dict of a C4-shaped run (10k contigs, 5M pairs); for each the SHA-1 of the three
    statistics files and the peak device memory of the first call above what was allocated before it, in torch's caching
    allocator and in the library's stream-ordered pool (its allocations under 32 MB; larger ones come from the library's
    workspace cache and are not counted); plus the device ranking and best-group kernels alone.

    python scripts/gfa_probe.py [--contigs 50000] [--pairs 200000000] [--reps 5] [--out gfa_probe.json]

Prints one JSON line (also written to --out) with the card name and power limit."""

import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TITLES = ("Link_threshold", "Link_density_threshold", "Link_density_ratio_threshold")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as exc:          # the numbers are still reported, with the failure instead of the card
        return "unknown ({})".format(exc)


class PoolUse:
    """Bytes in use in the device's default memory pool (where the library's cudaMallocAsync allocations under 32 MB live),
    with its high-water mark reset by ``start``."""
    USED_MEM_CURRENT, USED_MEM_HIGH = 7, 8          # CUmemPool_attribute

    def __init__(self, device):
        self.cu = ctypes.CDLL("libcuda.so.1")
        dev, self.pool = ctypes.c_int(), ctypes.c_void_p()
        for rc in (self.cu.cuInit(0), self.cu.cuDeviceGet(ctypes.byref(dev), device),
                   self.cu.cuDeviceGetDefaultMemPool(ctypes.byref(self.pool), dev)):
            if rc:
                raise RuntimeError("CUDA driver call failed: {}".format(rc))

    def _attr(self, attr):
        v = ctypes.c_uint64()
        if self.cu.cuMemPoolGetAttribute(self.pool, attr, ctypes.byref(v)):
            raise RuntimeError("cuMemPoolGetAttribute failed")
        return int(v.value)

    def start(self):
        zero = ctypes.c_uint64(0)
        if self.cu.cuMemPoolSetAttribute(self.pool, self.USED_MEM_HIGH, ctypes.byref(zero)):
            raise RuntimeError("cuMemPoolSetAttribute failed")
        return self._attr(self.USED_MEM_CURRENT)

    def high(self):
        return self._attr(self.USED_MEM_HIGH)


def time_statistics(cluster, fa_dict, links, groups, reps, pool, torch, dev):
    """Median seconds of one inflation's output_statistics over ``reps`` calls after a warm-up call, the SHA-1 of its three
    files, and the peak device bytes of the warm-up call above what was allocated before it (see PoolUse)."""
    t = []
    for rep in range(reps + 1):
        if rep == 0:
            torch.cuda.synchronize(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            torch_before, pool_before = torch.cuda.memory_allocated(dev), pool.start() if pool else None
        t0 = time.perf_counter()
        cluster.output_statistics(fa_dict, links, [(1, groups)])
        if rep:
            t.append(time.perf_counter() - t0)
        else:
            torch.cuda.synchronize(dev)
            peak = dict(pool_under_32mb=pool.high() - pool_before if pool else None,
                        torch=torch.cuda.max_memory_allocated(dev) - torch_before)
    sha = {}
    for title in TITLES:
        with open("inflation_1/{}_statistics.txt".format(title), "rb") as f:
            sha[title] = hashlib.sha1(f.read()).hexdigest()
    return dict(median_s=float(np.median(t)), min_s=float(min(t)), max_s=float(max(t)), sha1=sha, peak_device_bytes=peak)


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
    from tests.stats_oracle import reduce_phasing
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
        t0 = time.perf_counter()
        arr = reduce_phasing(cluster.LinkArrays(names, f["key_i"], f["key_j"], f["full"]), hap, w)
        res["full_link_reduction_s_w{}".format(w)] = dict(device_median=float(np.median(dev_s)), device_min=float(min(dev_s)),
                                                          host=time.perf_counter() - t0)
        res["full_links_after_w{}".format(w)] = len(arr)
        assert len(phased[w]) == len(arr) and np.array_equal(phased[w].values.astype(np.float64), arr.values.astype(np.float64))
    table.close()
    del f

    # the reference's dict of a C4-shaped run (10k contigs, 5M pairs, int values)
    asm4 = synth.make_assembly(a.nchr, 10000, 20000, seed=77)
    names4 = list(asm4.names)
    table4 = LinkTable(ctx, asm4.lengths, name_rank(names4), np.ones(asm4.n, np.uint8), 500 * 1000)
    table4.add(synth.make_pairs(asm4, 5_000_000, seed=78, device=dev))
    f4 = table4.fetch()
    table4.close()
    dict4 = cluster.LinkArrays(names4, f4["key_i"], f4["key_j"], f4["full"]).to_dict()
    fa4 = {n: [None, int(ln), 10] for n, ln in zip(names4, asm4.lengths.tolist())}
    per4 = asm4.n // a.nchr
    groups4 = [([names4[c] for c in range(g * per4, (g + 1) * per4)], 0) for g in range(a.nchr)]
    res["c4_dict_entries"] = len(dict4)

    # statistics of one inflation
    try:
        pool = PoolUse(ctx.device)
    except (OSError, AttributeError, RuntimeError) as exc:    # the times and digests are still reported
        pool, res["pool_error"] = None, str(exc)
    arr = phased[0.5]
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            os.makedirs("inflation_1", exist_ok=True)
            for tag, fa, links, grp in (("int", fa_dict, base, groups), ("float", fa_dict, arr, groups),
                                        ("c4_dict", fa4, dict4, groups4)):
                res["statistics_" + tag] = time_statistics(cluster, fa, links, grp, a.reps, pool, torch, dev)
        finally:
            os.chdir(cwd)
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
