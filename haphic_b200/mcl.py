"""Host side of the Markov-cluster path (hh_mcl handle).

Mirrors ``run_mcl_clustering`` / ``mcl`` / ``interpret_result``
(scripts/HapHiC_cluster.py:2026-2095, 2132-2162); the matrix work runs on the GPU.
"""

from __future__ import annotations

import ctypes as C
from decimal import Decimal

import numpy as np

from ._lib import HH_PREEXP_AUTO, HH_PREEXP_DENSE, HH_PREEXP_SPARSE, MclResult, MclStepInfo, PreexpInfo, check, load, ptr
from .links import LinkMatrix


class Mcl:
    """M0 = column-normalised link matrix and M1 = M0^expansion resident on the device, shared
    by every inflation of the sweep (HapHiC_cluster.py:2144-2158)."""

    PREEXP = {"auto": HH_PREEXP_AUTO, "sparse": HH_PREEXP_SPARSE, "dense": HH_PREEXP_DENSE}
    _close_order = 2

    def __init__(self, matrix: LinkMatrix, expansion: int = 2, col_lo: int = 0, col_hi: int | None = None,
                 preexp: str = "auto"):
        self.ctx = matrix.ctx
        self.n = matrix.n
        self.col_lo = int(col_lo)
        self.col_hi = self.n if col_hi is None else int(col_hi)
        self._own = (self.col_lo, self.col_hi)
        self._h = C.c_void_p()
        check(load().hh_mcl_create_ex(matrix._h, int(expansion), self.col_lo, self.col_hi, self.PREEXP[preexp],
                                      C.byref(self._h)))
        self.ctx.adopt(self)
        n = C.c_int32()
        nnz0 = C.c_int64()
        pre = C.c_int64()
        t0, t1 = C.c_float(), C.c_float()
        check(load().hh_mcl_info(self._h, C.byref(n), C.byref(nnz0), C.byref(pre), C.byref(t0), C.byref(t1)))
        self.nnz_m0 = int(nnz0.value)
        self.preexp_products = int(pre.value)
        self.normalize_ms, self.preexp_ms = float(t0.value), float(t1.value)
        pi = PreexpInfo()
        check(load().hh_mcl_preexp_info(self._h, C.byref(pi)))
        self.preexp = {k: getattr(pi, k) for k, _t in PreexpInfo._fields_}
        self.preexp["mode"] = {HH_PREEXP_SPARSE: "sparse", HH_PREEXP_DENSE: "dense"}.get(pi.mode, "?")
        self.last = None

    # -- inspection (parity tests) ------------------------------------------------------------
    def _fetch_csc(self, fn):
        import scipy.sparse as sp
        indptr = np.empty(self.n + 1, np.int64)
        check(fn(self._h, ptr(indptr), None, None))
        nnz = int(indptr[-1])
        indices = np.empty(nnz, np.int32)
        data = np.empty(nnz, np.float32)
        check(fn(self._h, ptr(indptr), ptr(indices), ptr(data)))
        return sp.csc_matrix((data, indices, indptr), shape=(self.n, self.n))

    def m0(self):
        return self._fetch_csc(load().hh_mcl_fetch_m0)

    def m1(self, col_lo: int | None = None, col_hi: int | None = None) -> np.ndarray:
        """Columns [col_lo, col_hi) of the pre-expanded matrix (default: the owned block), dense [n, col_hi-col_lo]
        (column-major on device)."""
        lo = self._own[0] if col_lo is None else int(col_lo)
        hi = self._own[1] if col_hi is None else int(col_hi)
        buf = np.empty((max(hi - lo, 0), self.n), np.float32)
        check(load().hh_mcl_fetch_m1_cols(self._h, lo, hi, ptr(buf)))
        return buf.T

    # -- one mcl() call on a single GPU ----------------------------------------------------------
    def run(self, inflation: float, max_iter: int = 200, pruning: float = 1e-4) -> dict:
        res = MclResult()
        it_nnz = np.zeros(max_iter, np.int64)
        it_prod = np.zeros(max_iter, np.int64)
        it_delta = np.zeros(max_iter, np.float32)
        it_ms = np.zeros(max_iter, np.float32)
        check(load().hh_mcl_run(self._h, float(inflation), int(max_iter), float(pruning), C.byref(res), ptr(it_nnz),
                                ptr(it_prod), ptr(it_delta), ptr(it_ms)))
        r = int(res.rounds)
        self.last = {
            "rounds": r, "converged": bool(res.converged), "nnz": int(res.nnz), "products": int(res.products),
            "bytes": int(res.bytes), "iter_nnz": it_nnz[:r].copy(), "iter_products": it_prod[:r].copy(),
            "iter_delta": it_delta[:r].copy(), "iter_ms": it_ms[:r].copy(),
        }
        return self.last

    def result(self):
        """The matrix the last run / committed step left, canonical CSC on the host."""
        return self._fetch_csc(load().hh_mcl_fetch_result)

    # -- step interface (column shards) -------------------------------------------------------
    def begin(self, inflation: float, pruning: float = 1e-4):
        check(load().hh_mcl_begin(self._h, float(inflation), float(pruning)))
        self.col_lo, self.col_hi = self._own

    def step(self, it: int):
        nnz = C.c_int64()
        prod = C.c_int64()
        delta = C.c_float()
        ms = C.c_float()
        check(load().hh_mcl_step(self._h, int(it), C.byref(nnz), C.byref(prod), C.byref(delta), C.byref(ms)))
        self.last_step_ms = float(ms.value)
        return int(nnz.value), int(prod.value), float(delta.value)

    def step_info(self) -> dict:
        """Engines the last step ran (hh_mcl_step_info): iteration 0 stream, block GEMM, window / small / column kernels."""
        si = MclStepInfo()
        check(load().hh_mcl_step_info(self._h, C.byref(si)))
        return {k: getattr(si, k) for k, _t in MclStepInfo._fields_}

    def pack(self, nnz_owned: int):
        """Owned block of the pending iterate as CUDA tensors (len int32 [ncols], idx int32, val fp32)."""
        import torch
        dev = torch.device("cuda", self.ctx.device)
        ncols = self.col_hi - self.col_lo
        ln = torch.empty(ncols, dtype=torch.int32, device=dev)
        idx = torch.empty(max(nnz_owned, 1), dtype=torch.int32, device=dev)
        val = torch.empty(max(nnz_owned, 1), dtype=torch.float32, device=dev)
        check(load().hh_mcl_pack(self._h, ptr(ln), ptr(idx), ptr(val)))
        return ln, idx[:nnz_owned], val[:nnz_owned]

    def pack_flat(self, nnz_owned: int, capacity: int):
        """The same three arrays laid out back to back in ONE int32 CUDA tensor of `capacity` words
        ([ncols] lengths, [nnz] row indices, [nnz] fp32 bit patterns): one collective moves a whole block."""
        import torch
        dev = torch.device("cuda", self.ctx.device)
        ncols = self.col_hi - self.col_lo
        buf = torch.empty(max(int(capacity), ncols + 2 * nnz_owned, 1), dtype=torch.int32, device=dev)
        base = buf.data_ptr()
        check(load().hh_mcl_pack(self._h, C.c_void_p(base), C.c_void_p(base + 4 * ncols), C.c_void_p(base + 4 * (ncols + nnz_owned))))
        return buf

    def unpack(self, col_lo: int, col_hi: int, ln, idx, val):
        check(load().hh_mcl_unpack(self._h, int(col_lo), int(col_hi), ptr(ln), ptr(idx), ptr(val), int(idx.shape[0])))

    def commit(self):
        check(load().hh_mcl_commit(self._h))

    def set_block(self, col_lo: int, col_hi: int):
        """Columns the following sparse steps compute (reset by begin())."""
        check(load().hh_mcl_set_block(self._h, int(col_lo), int(col_hi)))
        self.col_lo, self.col_hi = int(col_lo), int(col_hi)

    def close(self):
        if self._h:
            load().hh_mcl_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


GEMM_TILE = 128       # column tile of the pre-expansion GEMM: block boundaries fall on its multiples


def resolve_preexp(matrix: LinkMatrix, expansion: int, preexp: str = "auto") -> str:
    """The pre-expansion engine hh_mcl_create_ex would pick now ("sparse" or "dense")."""
    mode = C.c_int()
    check(load().hh_mcl_choose_preexp(matrix._h, int(expansion), Mcl.PREEXP[preexp], C.byref(mode)))
    return {HH_PREEXP_SPARSE: "sparse", HH_PREEXP_DENSE: "dense"}[mode.value]


def footprint(matrix: LinkMatrix, expansion: int, ncols: int, mode: str, pruning: float = 1e-4):
    """(M1 block bytes, bytes independent of ncols) an engine owning `ncols` columns holds on the device."""
    m1, fixed = C.c_size_t(), C.c_size_t()
    check(load().hh_mcl_footprint(matrix._h, int(expansion), int(ncols), Mcl.PREEXP[mode], float(pruning), C.byref(m1),
                                  C.byref(fixed)))
    return int(m1.value), int(fixed.value)


def available_bytes(ctx) -> int:
    """Device memory the next engine can allocate: free memory plus the library's idle cached blocks."""
    b = C.c_size_t()
    check(load().hh_ctx_mem_available(ctx.handle, C.byref(b)))
    return int(b.value)


def plan_column_blocks(n: int, footprint, budget: int, tile: int = GEMM_TILE):
    """Contiguous column blocks [(lo, hi)] covering [0, n), as few as possible, each with sum(footprint(hi - lo)) <= budget.
    Every boundary but n is a multiple of `tile`.  footprint(ncols) -> (M1 block bytes, fixed bytes), non-decreasing in ncols."""
    def fits(w):
        return sum(footprint(w)) <= budget

    if fits(n):
        return [(0, n)]
    if not fits(min(tile, n)):
        m1, fixed = footprint(min(tile, n))
        raise MemoryError("Markov clustering needs {} bytes of device memory for one {}-column block of the pre-expanded "
                          "matrix plus {} bytes that do not depend on the block; {} bytes are available".format(
                              m1, min(tile, n), fixed, budget))

    def widest(lo, hi, step):           # largest w in {lo, lo + step, ..., <= hi} that fits (lo fits)
        a, b = lo // step, hi // step
        while a < b:
            mid = (a + b + 1) // 2
            if fits(mid * step):
                a = mid
            else:
                b = mid - 1
        return a * step

    w = widest(tile, n, tile)           # aligned blocks
    last = widest(w, n, 1)              # the last block ends at n and need not be aligned
    k = 1 + -(-(n - last) // w)
    return [(i * w, (i + 1) * w) for i in range(k - 1)] + [((k - 1) * w, n)]


def continue_from_iteration0(engine, inflation: float, pruning: float, max_iter: int, n: int, others, first):
    """The rest of one mcl() call once iteration 0 of every column block exists: iteration 0 of the engine's own block
    again, the other blocks unpacked (`others` yields (lo, hi, lengths, row indices, values) device tensors), and the
    remaining iterations with every column owned -- the single-GPU code path.  `first` = (nnz, products, ms) of iteration 0
    over all columns.  Returns {"rounds", "converged", "iter_nnz", "iter_products", "iter_ms", "iter_delta"}."""
    engine.begin(inflation, pruning)
    engine.step(0)
    for lo, hi, ln, idx, val in others:
        engine.unpack(lo, hi, ln, idx, val)
    engine.commit()
    engine.set_block(0, n)
    st = {"rounds": 1, "converged": False, "iter_nnz": [first[0]], "iter_products": [first[1]], "iter_ms": [first[2]],
          "iter_delta": [0.0]}
    for it in range(1, max_iter):
        nnz, prod, delta = engine.step(it)
        engine.commit()
        st["iter_nnz"].append(nnz)
        st["iter_products"].append(prod)
        st["iter_ms"].append(getattr(engine, "last_step_ms", 0.0))
        st["iter_delta"].append(delta)
        st["rounds"] = it + 1
        if it > 1 and delta <= 1e-8:
            st["converged"] = True
            break
    return st


def _run_stats(st, n: int) -> dict:
    """Statistics of continue_from_iteration0 in the form Mcl.run returns them (hh_mcl_run's byte count included)."""
    nnz = np.asarray(st["iter_nnz"], np.int64)
    moved = 4 * n * n + 8 * int(nnz[0]) + sum(16 * int(a) + 8 * int(b) + 12 * (n + 1) for a, b in zip(nnz[:-1], nnz[1:]))
    return {"rounds": st["rounds"], "converged": st["converged"], "nnz": int(nnz[-1]), "products": int(sum(st["iter_products"])),
            "bytes": moved, "iter_nnz": nnz, "iter_products": np.asarray(st["iter_products"], np.int64),
            "iter_delta": np.asarray(st["iter_delta"], np.float32), "iter_ms": np.asarray(st["iter_ms"], np.float32)}


def blocked_sweep(matrix: LinkMatrix, expansion: int, inflations, max_iter: int, pruning: float, mode: str, blocks,
                  engine_cls=Mcl, timing: dict | None = None):
    """An inflation sweep whose pre-expanded matrix M1 is never whole on the device.  Only iteration 0 of an mcl() call
    reads M1, and its columns are independent, so:
      phase A  one engine per column block in turn (M1 of that block only): iteration 0 of every inflation, the pruned
               block kept in pinned host memory; every engine but the last is closed before the next one is built;
      phase B  per inflation, the last block's engine rebuilds the whole iterate from the kept blocks and runs the
               remaining iterations owning every column (continue_from_iteration0).
    `mode` is the resolved engine ("sparse" / "dense"): every block must come from the same one.  Yields
    (inflation, statistics as Mcl.run returns them, engine holding the result) in sweep order.  `timing` (optional) gets
    the seconds of each phase and the device milliseconds of the pre-expansion over all blocks."""
    import time

    import torch
    n = matrix.n
    saved = [[] for _ in inflations]           # per inflation: (lo, hi, lengths, rows, values) of every block but the last
    first = [[0, 0, 0.0] for _ in inflations]
    engine = None
    t0 = time.perf_counter()
    try:
        for b, (lo, hi) in enumerate(blocks):
            if engine is not None:
                engine.close()
                engine = None
                if torch.cuda.is_available():
                    torch.cuda.empty_cache()   # the packed blocks went through torch's allocator: give the memory back
            engine = engine_cls(matrix, expansion, lo, hi, preexp=mode)
            if timing is not None:
                timing["preexp_ms"] = timing.get("preexp_ms", 0.0) + getattr(engine, "preexp_ms", 0.0)
            for k, r in enumerate(inflations):
                engine.begin(float(r), pruning)
                nnz, prod, _delta = engine.step(0)
                first[k][0] += nnz
                first[k][1] += prod
                first[k][2] += getattr(engine, "last_step_ms", 0.0)
                if b + 1 < len(blocks):
                    host = []
                    for t in engine.pack(nnz):
                        h = torch.empty(t.shape, dtype=t.dtype, pin_memory=t.is_cuda)
                        h.copy_(t)
                        host.append(h)
                    saved[k].append((lo, hi, *host))
        if timing is not None:
            timing["phase_a_s"] = time.perf_counter() - t0
        dev = torch.device("cuda", engine.ctx.device) if getattr(engine, "ctx", None) is not None else torch.device("cpu")

        def uploaded(k):
            for lo, hi, ln, idx, val in saved[k]:
                yield lo, hi, ln.to(dev), idx.to(dev), val.to(dev)
            if dev.type == "cuda":
                torch.cuda.empty_cache()      # the uploads are unpacked: leave their memory to the iterations

        if timing is not None:
            timing["phase_b_s"] = 0.0
        for k, r in enumerate(inflations):
            t1 = time.perf_counter()
            st = continue_from_iteration0(engine, float(r), pruning, max_iter, n, uploaded(k), first[k])
            saved[k] = None
            if timing is not None:
                timing["phase_b_s"] += time.perf_counter() - t1
            yield r, _run_stats(st, n), engine
    finally:
        if engine is not None:
            engine.close()


def interpret_result(result):
    """Attractor rows -> clusters (HapHiC_cluster.py:2065-2095).  ``result`` is a scipy sparse
    matrix; returns a list of index tuples, or None when a node is in two clusters or in none."""
    import scipy.sparse as sp
    r = sp.csr_matrix(result)
    r.eliminate_zeros()
    r.sort_indices()
    n = r.shape[0]
    attractors = np.nonzero(r.diagonal())[0]
    clusters = set()
    for a in attractors.tolist():
        clusters.add(tuple(r.indices[r.indptr[a]:r.indptr[a + 1]].tolist()))
    seen = np.zeros(n, dtype=np.int64)
    for c in clusters:
        np.add.at(seen, list(c), 1)
    if n == 0 or seen.min() != 1 or seen.max() != 1:
        return None
    return list(clusters)


def inflation_values(min_inflation, max_inflation, step):
    """The Decimal sweep of run_mcl_clustering (2139-2141, 2155); ``str(v)`` names the output dirs."""
    start = Decimal(str(min_inflation))
    st = Decimal(str(step))
    end = Decimal(str(max_inflation)) + st
    import math
    n = max(0, math.ceil((end - start) / st))       # numpy.arange length rule, exact in Decimal
    # numpy.arange over Decimals: element 0 is `start` itself ('1.0', not '1.00'), element k is start + k * step
    return [start if k == 0 else start + k * st for k in range(n)]
