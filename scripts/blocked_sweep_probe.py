"""Blocked Markov-clustering sweep on one GPU (haphic_b200.mcl.blocked_sweep): wall time of phase A (iteration 0 of every
inflation per column block of M1) and phase B (the rest of every mcl() call), and the pre-expansion device time summed
over the blocks.

  --c3      the benchmark's matrix (50k contigs / 200M pairs): the resident engine against 2 and 4 forced blocks,
            alternated in one process (rounds of the three arms, medians reported)
  --c5      150k contigs / 32 chromosomes / 300M pairs with the budget the CLI uses: blocks, peak device memory sampled
            every 20 ms, phase times, and the checks of tests/test_gpu_mcl_blocked.py
  --resident-only   (with --c5) just try the resident engine on the C5 matrix and report how it ends

Writes one JSON line per measurement to stdout and to --out."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


class MemSampler:
    """Lowest free device memory seen (torch.cuda.mem_get_info every 20 ms on a host thread)."""

    def __init__(self):
        import torch
        self.torch = torch
        self.total = torch.cuda.mem_get_info()[1]
        self.min_free = self.total
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            self.min_free = min(self.min_free, self.torch.cuda.mem_get_info()[0])
            time.sleep(0.02)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    @property
    def peak_used(self):
        return self.total - self.min_free


def link_matrix(ctx, nchr, n_contigs, mean_len, n_pairs, seed):
    from haphic_b200 import synth
    from haphic_b200.links import LinkTable, name_rank
    asm = synth.make_assembly(nchr, n_contigs, mean_len, seed=seed)
    rank = name_rank(asm.names)
    in_nx = np.ones(asm.n, np.uint8)
    rec = synth.make_pairs_range(asm, 0, n_pairs, seed=seed + 1, device="cuda")
    tab = LinkTable(ctx, asm.lengths, rank, in_nx, 500000, capacity_hint=int(0.45 * n_pairs))
    tab.add(rec, asynchronous=True)
    tab.finish()
    del rec
    keep = np.ones(asm.n, np.uint8)
    index, n_linked = tab.linked_index(keep)
    tail = np.nonzero(index < 0)[0].astype(np.int32)
    mat = tab.to_matrix(keep, tail)
    tab.close()
    ctg_of = np.empty(mat.n, np.int64)
    ctg_of[index[index >= 0]] = np.nonzero(index >= 0)[0]
    ctg_of[n_linked + np.arange(len(tail))] = tail
    import torch
    torch.cuda.empty_cache()
    return asm, mat, ctg_of


def emit(out, rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def resident_arm(mat, mode, inflations):
    from haphic_b200.mcl import Mcl
    t0 = time.perf_counter()
    eng = Mcl(mat, 2, preexp=mode)
    eng.ctx.sync()
    t1 = time.perf_counter()
    stats = []
    for r in inflations:
        st = eng.run(r, 200, 1e-4)
        eng.result()
        stats.append((st["rounds"], st["iter_nnz"].tolist()))
    t2 = time.perf_counter()
    pre = eng.preexp_ms
    eng.close()
    return {"phase_a_s": t1 - t0, "phase_b_s": t2 - t1, "preexp_ms": pre}, stats


def blocked_arm(mat, mode, inflations, blocks):
    from haphic_b200.mcl import blocked_sweep
    timing = {}
    stats = []
    for _r, st, eng in blocked_sweep(mat, 2, inflations, 200, 1e-4, mode, blocks, timing=timing):
        eng.result()
        stats.append((st["rounds"], st["iter_nnz"].tolist()))
    return timing, stats


def c3(a):
    from haphic_b200._lib import Context
    from haphic_b200.mcl import footprint, plan_column_blocks, resolve_preexp
    inflations = [1.5, 2.0, 3.0]
    with Context(0) as ctx:
        _asm, mat, _ = link_matrix(ctx, 24, 50000, 20000, 200_000_000, 12345)
        n = mat.n
        mode = resolve_preexp(mat, 2, "auto")

        def plan(k):
            w = -(-(-(-n // k)) // 128) * 128
            return plan_column_blocks(n, lambda c: footprint(mat, 2, c, mode), sum(footprint(mat, 2, w, mode)))
        arms = {"resident": None, "blocks2": plan(2), "blocks4": plan(4)}
        res = {k: [] for k in arms}
        ref = None
        blocked_arm(mat, mode, inflations, arms["blocks2"])           # warm-up of every kernel shape
        for rep in range(a.reps):
            for name, blocks in arms.items():
                t, stats = resident_arm(mat, mode, inflations) if blocks is None else blocked_arm(mat, mode, inflations, blocks)
                ref = stats if ref is None else ref
                assert stats == ref, name                          # same rounds and entry counts as the resident run
                res[name].append(t)
        for name, ts in res.items():
            emit(a.out, {"probe": "c3", "card": card(), "arm": name, "mode": mode, "n": n, "inflations": inflations,
                         "blocks": arms[name] or [(0, n)], "reps": len(ts),
                         **{k: float(np.median([t[k] for t in ts])) for k in ("phase_a_s", "phase_b_s", "preexp_ms")},
                         "all": ts})
        mat.close()


def c5(a):
    import torch
    from haphic_b200._lib import Context
    from haphic_b200.cluster import _mcl_budget
    from haphic_b200.mcl import Mcl, available_bytes, blocked_sweep, footprint, interpret_result, plan_column_blocks, resolve_preexp
    inflations = [1.5, 2.0, 3.0]
    with Context(0) as ctx:
        t0 = time.perf_counter()
        asm, mat, ctg_of = link_matrix(ctx, 32, 150000, 20000, 300_000_000, 12345)
        n = mat.n
        build_s = time.perf_counter() - t0
        mode = resolve_preexp(mat, 2, "auto")
        avail = available_bytes(ctx)
        m1_all, fixed = footprint(mat, 2, n, mode)
        base = {"probe": "c5", "card": card(), "n": n, "nnz": int(mat.nnz) if hasattr(mat, "nnz") else None, "mode": mode,
                "link_build_s": build_s, "available_bytes": avail, "m1_bytes": m1_all, "fixed_bytes": fixed}
        if a.resident_only:
            try:
                eng = Mcl(mat, 2)
                emit(a.out, dict(base, resident="created", preexp=eng.preexp["mode"]))
                eng.close()
            except Exception as exc:
                emit(a.out, dict(base, resident="failed", error=str(exc)))
            mat.close()
            return
        budget = _mcl_budget(ctx)
        blocks = plan_column_blocks(n, lambda w: footprint(mat, 2, w, mode), budget)
        chrom = asm.chrom[ctg_of]
        timing, per = {}, []
        with MemSampler() as ms:
            for r, st, eng in blocked_sweep(mat, 2, inflations, 200, 1e-4, mode, blocks, timing=timing):
                fin = eng.result()
                colsum = float(abs(np.asarray(fin.sum(axis=0)).ravel() - 1.0).max())
                cl = interpret_result(fin)
                pure = sum(int(np.bincount(chrom[list(c)]).max()) for c in cl) if cl else 0
                per.append({"inflation": r, "rounds": st["rounds"], "converged": st["converged"], "colsum_err": colsum,
                            "clusters": len(cl) if cl else None, "covered": sum(len(c) for c in cl) if cl else 0,
                            "pure_fraction": pure / n})
        emit(a.out, dict(base, budget=budget, blocks=blocks, peak_used_bytes=ms.peak_used, total_bytes=ms.total,
                         torch_reserved=torch.cuda.memory_reserved(), **timing, inflations=per))
        mat.close()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--c3", action="store_true")
    p.add_argument("--c5", action="store_true")
    p.add_argument("--resident-only", action="store_true")
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--out", default="")
    a = p.parse_args()
    if a.c3:
        c3(a)
    if a.c5:
        c5(a)


if __name__ == "__main__":
    main()
