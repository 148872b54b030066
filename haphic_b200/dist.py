"""Multi-GPU orchestration (one process per GPU, torch.distributed over NCCL/NVLink).

The path shards in two places (SURVEY.md section 8e):

* link counting -- the read-pair stream is cut into contiguous shards, one per rank; every record is
  routed to the rank that owns its contig pair (one all-to-all of records and stream indices), counted
  there into a partition table disjoint from every other rank's, and the compact partitions are
  all-gathered so each rank ends with the whole table (integer adds and mins: bit-identical for any
  world size).  `merge_link_tables` is the older exchange (count locally, all-gather tables, re-insert);
* Markov clustering -- every step of an iteration is column-local, so each rank owns a contiguous
  block of columns; per iteration there is ONE exchange, an all-gather of the pruned column blocks
  (lengths, then packed row indices and values), plus a scalar max for the convergence test.
  The dense pre-expanded matrix is never exchanged: each rank computes its own column block of it.

The exchange code is device-agnostic (it moves whatever torch tensors the engine hands it), which is
how the world_size-2 gloo tests exercise it on CPU.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.distributed as dist

from .mcl import continue_from_iteration0


def column_blocks(n: int, world: int):
    """Contiguous, near-equal column blocks [(lo, hi)] * world."""
    cuts = [(n * r) // world for r in range(world + 1)]
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def balanced_column_blocks(cost, world: int):
    """Contiguous blocks with near-equal total `cost` (e.g. per-column product estimates)."""
    c = np.asarray(cost, dtype=np.float64)
    n = len(c)
    if n == 0 or c.sum() <= 0:
        return column_blocks(n, world)
    cum = np.concatenate([[0.0], np.cumsum(c)])
    cuts = [0]
    for r in range(1, world):
        k = int(np.searchsorted(cum, cum[-1] * r / world))
        cuts.append(min(max(k, cuts[-1]), n))
    cuts.append(n)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def allgather_varlen(t: torch.Tensor, group=None):
    """All-gather 1-D (or [m, k]) tensors whose leading size differs per rank.
    Returns the list of every rank's tensor (this rank's own included)."""
    world = dist.get_world_size(group)
    m = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    sizes = [torch.zeros_like(m) for _ in range(world)]
    dist.all_gather(sizes, m, group=group)
    sizes = [int(s.item()) for s in sizes]
    mx = max(max(sizes), 1)
    pad_shape = (mx,) + tuple(t.shape[1:])
    padded = torch.zeros(pad_shape, dtype=t.dtype, device=t.device)
    padded[: t.shape[0]] = t
    outs = [torch.empty(pad_shape, dtype=t.dtype, device=t.device) for _ in range(world)]
    dist.all_gather(outs, padded, group=group)
    return [o[:s] for o, s in zip(outs, sizes)]


def _wait_collectives(t: torch.Tensor):
    """The library works on its own CUDA stream: make sure the collectives torch enqueued on its
    current stream have landed before a library kernel reads their output."""
    if t.is_cuda:
        torch.cuda.current_stream(t.device).synchronize()


def merge_link_tables(table, group=None):
    """Every rank holds a table with its own shard counted.  Afterwards every rank's table holds
    the whole stream (call table.finish() next).  One all-gather of the exported entries."""
    rank = dist.get_rank(group)
    world = dist.get_world_size(group)
    table.finish()
    ent, tot, n_rec, n_used = table.export()
    ents = allgather_varlen(ent, group)
    tots = [torch.empty_like(tot) for _ in range(world)]
    dist.all_gather(tots, tot, group=group)
    meta = torch.tensor([n_rec, n_used], dtype=torch.int64, device=ent.device)
    metas = [torch.zeros_like(meta) for _ in range(world)]
    dist.all_gather(metas, meta, group=group)
    _wait_collectives(ent)
    for r in range(world):
        if r == rank:
            continue
        table.merge(ents[r], tots[r], int(metas[r][0].item()), int(metas[r][1].item()))


REPLICATE_BELOW = 8      # entries per column under which column shards stop exchanging (see sharded_mcl_run)


def routed_link_build(table, rec, stream_lo: int, group=None):
    """Sharded link counting without a reduction (SURVEY.md 8e): every rank holds a contiguous shard `rec` of the
    read stream (global index of rec[0] = stream_lo).  Records are routed to the rank that owns their contig pair
    (one all-to-all of records + stream indices), counted there into disjoint partition tables, and the compact
    partitions are all-gathered so that every rank ends with the whole table (unordered until somebody fetches it).
    Returns the LinksInfo of the whole table."""
    rank = dist.get_rank(group)
    world = dist.get_world_size(group)
    dbg = os.environ.get("HH_BENCH_DEBUG") == "2"
    marks = []

    def mark(tag):
        if dbg:
            import time
            torch.cuda.synchronize()
            marks.append((tag, time.perf_counter()))
    mark("start")
    rec_out, pos_out, counts = table.route(rec, stream_lo, world)
    mark("route")
    dev = rec_out.device
    send = torch.tensor(counts, dtype=torch.int64, device=dev)
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)
    recv_counts = [int(x) for x in recv.tolist()]
    rec_in = torch.empty((sum(recv_counts), 4), dtype=rec_out.dtype, device=dev)
    pos_in = torch.empty(sum(recv_counts), dtype=pos_out.dtype, device=dev)
    dist.all_to_all_single(rec_in, rec_out, recv_counts, counts, group=group)
    dist.all_to_all_single(pos_in, pos_out, recv_counts, counts, group=group)
    _wait_collectives(rec_in)
    mark("all-to-all")
    table.add_routed(rec_in, pos_in)
    del rec_out, pos_out
    part = table.finish_partition()
    ent, tot, _, _ = table.export()
    mark("insert+partition+export")
    # sizes, then the partitions straight into one buffer (uneven all-gather)
    meta = torch.tensor([int(ent.shape[0]), int(rec.shape[0]), int(part.n_used), int(stream_lo) + int(rec.shape[0])],
                        dtype=torch.int64, device=dev)
    metas = [torch.empty_like(meta) for _ in range(world)]
    dist.all_gather(metas, meta, group=group)
    metas = [m.tolist() for m in metas]
    sizes = [int(m[0]) for m in metas]
    whole = torch.empty((sum(sizes), 9), dtype=ent.dtype, device=dev)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    if len(set(sizes)) == 1:
        dist.all_gather_into_tensor(whole.view(-1), ent.reshape(-1), group=group)
    else:
        # uneven partitions (the usual case: pairs are split by a hash): ONE all-gather of blocks padded to the largest, then a
        # device-side compaction -- eight broadcasts in a row cost more than the padding
        cap = max(sizes)
        mine = torch.empty((cap, 9), dtype=ent.dtype, device=dev)
        mine[: sizes[rank]].copy_(ent)
        padded = torch.empty((world, cap, 9), dtype=ent.dtype, device=dev)
        dist.all_gather_into_tensor(padded.view(-1), mine.view(-1), group=group)
        _wait_collectives(padded)
        for r in range(world):
            whole[int(offs[r]):int(offs[r + 1])].copy_(padded[r, : sizes[r]])
        del padded, mine
    dist.all_reduce(tot, op=dist.ReduceOp.SUM, group=group)
    _wait_collectives(whole)
    mark("all-gather")
    info = table.adopt(whole, tot, sum(int(m[1]) for m in metas), sum(int(m[2]) for m in metas), max(int(m[3]) for m in metas))
    mark("adopt")
    if dbg:
        print("rank", rank, "routed build ms:", [(b[0], round(1000 * (b[1] - a[1]), 1)) for a, b in zip(marks, marks[1:])],
              file=sys.stderr, flush=True)
    return info


def sharded_mcl_run(engine, inflation: float, max_iter: int, pruning: float, blocks, group=None):
    """One mcl() call (HapHiC_cluster.py:2026-2062) over column shards.

    `engine` owns the block blocks[rank] and offers begin / step / pack / unpack / commit
    (haphic_b200.mcl.Mcl, or a CPU stand-in in the gloo tests).  Returns
    {"rounds", "converged", "iter_nnz", "iter_products"} identical on every rank."""
    rank = dist.get_rank(group)
    world = dist.get_world_size(group)
    engine.begin(inflation, pruning)
    rounds, converged = 0, False
    it_nnz, it_prod, it_ms = [], [], []
    ncols = [hi - lo for lo, hi in blocks]
    n_total = blocks[-1][1]
    replicated = False
    for it in range(max_iter):
        nnz, prod, delta = engine.step(it)
        if replicated:
            # every rank computes the whole (tiny) iterate itself: identical on all ranks, nothing to exchange
            engine.commit()
            it_nnz.append(nnz)
            it_prod.append(prod)
            it_ms.append(getattr(engine, "last_step_ms", 0.0))
            rounds = it + 1
            if it > 1 and delta <= 1e-8:
                converged = True
                break
            continue
        # exchange 1 (tiny): every rank's nnz / products / convergence term -> sizes of the blocks and the statistics
        dev = engine_device(engine)
        meta = torch.tensor([float(nnz), float(prod), float(delta)], dtype=torch.float64, device=dev)
        metas = torch.empty(world * 3, dtype=torch.float64, device=dev)
        dist.all_gather_into_tensor(metas, meta, group=group)
        metas = metas.view(world, 3).tolist()
        nnzs = [int(m[0]) for m in metas]
        cap = max(c + 2 * z for c, z in zip(ncols, nnzs))
        # exchange 2: the packed blocks ([lengths | row indices | value bits], padded to the largest), one all-gather
        if hasattr(engine, "pack_flat"):
            buf = engine.pack_flat(nnz, cap)
        else:
            ln, idx, val = engine.pack(nnz)
            buf = torch.zeros(cap, dtype=torch.int32, device=dev)
            buf[: ncols[rank]] = ln
            buf[ncols[rank]: ncols[rank] + nnz] = idx
            buf[ncols[rank] + nnz: ncols[rank] + 2 * nnz] = val.view(torch.int32)
        out = torch.empty(world * cap, dtype=torch.int32, device=dev)
        dist.all_gather_into_tensor(out, buf[:cap], group=group)
        _wait_collectives(out)
        out = out.view(world, cap)
        for r in range(world):
            if r != rank:
                c, z = ncols[r], nnzs[r]
                engine.unpack(blocks[r][0], blocks[r][1], out[r, :c], out[r, c: c + z], out[r, c + z: c + 2 * z].view(torch.float32))
        engine.commit()
        if world > 1 and it >= 1 and sum(nnzs) <= REPLICATE_BELOW * n_total and hasattr(engine, "set_block"):
            engine.set_block(0, n_total)     # nearly converged: a full step costs less than one exchange
            replicated = True
        it_nnz.append(sum(nnzs))
        it_prod.append(sum(int(m[1]) for m in metas))
        it_ms.append(getattr(engine, "last_step_ms", 0.0))
        rounds = it + 1
        if it > 1 and max(m[2] for m in metas) <= 1e-8:
            converged = True
            break
    return {"rounds": rounds, "converged": converged, "iter_nnz": it_nnz, "iter_products": it_prod, "iter_ms": it_ms}


def sharded_mcl_sweep(engine, inflations, max_iter: int, pruning: float, blocks, group=None, on_result=None):
    """The inflation sweep of run_mcl_clustering (HapHiC_cluster.py:2155-2158) over column shards, inflation-parallel.

    Only iteration 0 of an mcl() call touches the dense pre-expanded matrix, which is what the ranks shard.  So:
      phase A  every rank runs iteration 0 of EVERY inflation on its column block and the pruned blocks are all-gathered
               (one collective per inflation, kept as packed buffers);
      phase B  inflation k belongs to rank k mod world, which rebuilds the whole iterate from the saved buffers and runs the
               remaining iterations alone as the owner of every column -- exactly the single-GPU code path (component blocks
               on the tensor cores included), no further exchange.
    `on_result(k, inflation, engine)` is called on the owner right after inflation k has finished (fetch / write its result
    there).  Returns the list of per-inflation statistics, identical on every rank."""
    rank = dist.get_rank(group)
    world = dist.get_world_size(group)
    if world == 1 or not hasattr(engine, "set_block"):
        out = []
        for k, r in enumerate(inflations):
            st = sharded_mcl_run(engine, r, max_iter, pruning, blocks, group=group)
            st["owner"] = 0
            out.append(st)
            if on_result is not None and rank == 0:
                on_result(k, r, engine)
        return out
    dev = engine_device(engine)
    ncols = [hi - lo for lo, hi in blocks]
    n_total = blocks[-1][1]
    saved = []
    for r in inflations:                                             # ---- phase A
        engine.begin(r, pruning)
        nnz, prod, _delta = engine.step(0)
        meta = torch.tensor([float(nnz), float(prod)], dtype=torch.float64, device=dev)
        metas = torch.empty(world * 2, dtype=torch.float64, device=dev)
        dist.all_gather_into_tensor(metas, meta, group=group)
        metas = metas.view(world, 2).tolist()
        nnzs = [int(m[0]) for m in metas]
        cap = max(c + 2 * z for c, z in zip(ncols, nnzs))
        if hasattr(engine, "pack_flat"):
            buf = engine.pack_flat(nnz, cap)
        else:
            ln, idx, val = engine.pack(nnz)
            buf = torch.zeros(cap, dtype=torch.int32, device=dev)
            buf[: ncols[rank]] = ln
            buf[ncols[rank]: ncols[rank] + nnz] = idx
            buf[ncols[rank] + nnz: ncols[rank] + 2 * nnz] = val.view(torch.int32)
        out = torch.empty(world * cap, dtype=torch.int32, device=dev)
        dist.all_gather_into_tensor(out, buf[:cap], group=group)
        _wait_collectives(out)
        saved.append((out.view(world, cap), nnzs, sum(int(m[1]) for m in metas), getattr(engine, "last_step_ms", 0.0)))
    local = {}
    for k, r in enumerate(inflations):                               # ---- phase B
        if k % world != rank:
            saved[k] = None
            continue
        out, nnzs, prod0, ms0 = saved[k]
        # this rank's own block again (a 1/world stream of M1), then the others' from the saved buffers
        others = ((blocks[rr][0], blocks[rr][1], out[rr, :ncols[rr]], out[rr, ncols[rr]: ncols[rr] + nnzs[rr]],
                   out[rr, ncols[rr] + nnzs[rr]: ncols[rr] + 2 * nnzs[rr]].view(torch.float32)) for rr in range(world) if rr != rank)
        st = continue_from_iteration0(engine, r, pruning, max_iter, n_total, others, (sum(nnzs), prod0, ms0))
        st["owner"] = rank
        local[k] = st
        if on_result is not None:
            on_result(k, r, engine)
        saved[k] = None
    gathered = [None] * world
    dist.all_gather_object(gathered, local, group=group)
    merged = {}
    for g in gathered:
        merged.update(g)
    return [merged[k] for k in range(len(inflations))]


def engine_device(engine):
    ctx = getattr(engine, "ctx", None)
    return torch.device("cuda", ctx.device) if ctx is not None else torch.device("cpu")


def _equal_blocks(blocks):
    return len({hi - lo for lo, hi in blocks}) == 1


def _gather_lens(lens, ln, blocks, group):
    got = allgather_varlen(ln, group)
    for r in range(len(blocks)):
        lens[r] = got[r]


# ------------------------------------------------------------------------------------------------
# bench.py --gpus N (launched by torch.distributed.run, one rank per GPU)
# ------------------------------------------------------------------------------------------------

def rank0_roofline(s):
    """Rank 0's pre-expansion launch (its column block of M0*M0), same definitions as the single-GPU line."""
    import bench as B
    return B.preexp_roofline(s["preexp"], s["n_matrix"], s["nnz_m0"], s["own_cols"], {})


def bench_multi(a, world: int, rank_id: int, local: int):
    import json
    import time

    import bench as B
    from ._lib import Context
    from .links import LinkTable
    from .mcl import Mcl

    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    inflations = [float(x) for x in a.inflations.split(",")]
    asm, rank, in_nx, rec, stream_lo = B.make_inputs(a, dev, rank_id, world)
    n = asm.n
    P_local = int(rec.shape[0])
    keep = np.ones(n, np.uint8)
    ctx = Context(local)
    stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
    hint = int(min(a.pairs, n * (n - 1) // 2) * (0.45 if a.pairs > 4_000_000 else 1.0) / world * 1.1)   # one partition

    def barrier():
        dist.barrier()
        torch.cuda.synchronize()

    def one_step():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        barrier()
        ev[0].record(stream)
        tab = LinkTable(ctx, asm.lengths, rank, in_nx, 500000, capacity_hint=hint)
        info = routed_link_build(tab, rec, stream_lo)
        index, n_linked = tab.linked_index(keep)
        mat = tab.to_matrix(keep, np.nonzero(index < 0)[0].astype(np.int32))
        ev[1].record(stream)
        blocks = column_blocks(mat.n, world)
        mc = Mcl(mat, col_lo=blocks[rank_id][0], col_hi=blocks[rank_id][1])
        tw = time.perf_counter()
        stats = sharded_mcl_sweep(mc, inflations, a.max_iter, a.pruning, blocks)
        iters = sum(st["rounds"] for st in stats)
        if os.environ.get("HH_BENCH_DEBUG") and rank_id == 0:
            print("mcl sweep wall_ms={:.1f} preexp={:.1f} norm={:.1f}".format(1000 * (time.perf_counter() - tw), mc.preexp_ms, mc.normalize_ms),
                  [(r, st["owner"], st["rounds"], round(sum(st["iter_ms"]), 1), [round(x, 1) for x in st["iter_ms"][:4]])
                   for r, st in zip(inflations, stats)], file=sys.stderr, flush=True)
        ev[2].record(stream)
        ev[2].synchronize()
        t = torch.tensor([ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)          # max over ranks
        out = {"build_ms": float(t[0].item()), "mcl_ms": float(t[1].item()), "iters": iters,
               "nnz_full": int(info.nnz_full), "n_matrix": mat.n, "preexp_ms": mc.preexp_ms, "nnz_m0": mc.nnz_m0,
               "own_cols": blocks[rank_id][1] - blocks[rank_id][0], "preexp_products": mc.preexp_products,
               "preexp": dict(mc.preexp)}
        mc.close()
        mat.close()
        tab.close()
        return out

    for _ in range(a.warmup):
        one_step()
    sampler = B.ClockSampler(local)
    if rank_id == 0:
        sampler.start()
    l0 = ctx.launches
    barrier()
    t0 = time.perf_counter()
    steps = [one_step() for _ in range(a.steps)]
    barrier()
    wall = time.perf_counter() - t0
    launches = ctx.launches - l0
    clocks = sampler.stop() if rank_id == 0 else None

    # ---- end to end: pinned HOST shard in, host results out on rank 0 (H2D / D2H inside the timed region)
    from .mcl import interpret_result
    if a.e2e_steps > 0:
        rec_host = torch.empty(rec.shape, dtype=torch.int32, pin_memory=True)
        rec_host.copy_(rec)
    torch.cuda.synchronize()
    e2e_t, d2h = [], 0
    e2e_warm = 2            # pinned result buffers are allocated by the first pass, which also skews the second
    for s in range(e2e_warm + a.e2e_steps if a.e2e_steps > 0 else 0):
        barrier()
        t0 = time.perf_counter()
        tab = LinkTable(ctx, asm.lengths, rank, in_nx, 500000, capacity_hint=hint)
        dbg = [time.perf_counter()]
        rec_dev = rec_host.to(dev, non_blocking=True)       # H2D of this rank's shard, inside the timed region
        _wait_collectives(rec_dev)
        dbg.append(time.perf_counter())
        routed_link_build(tab, rec_dev, stream_lo)
        del rec_dev
        dbg.append(time.perf_counter())
        if rank_id == 0:
            table = tab.fetch(pinned=True)
            tot = tab.fetch_ctg()
        dbg.append(time.perf_counter())
        index, n_linked = tab.linked_index(keep)
        mat = tab.to_matrix(keep, np.nonzero(index < 0)[0].astype(np.int32))
        ctx.sync()
        dbg.append(time.perf_counter())
        barrier()
        t1 = time.perf_counter()
        if os.environ.get("HH_BENCH_DEBUG"):
            print("rank", rank_id, "e2e build sections ms (h2d, routed build, fetch, index+matrix):",
                  [round(1000 * (b - a_), 1) for a_, b in zip(dbg, dbg[1:])], file=sys.stderr, flush=True)
        blocks = column_blocks(mat.n, world)
        mc = Mcl(mat, col_lo=blocks[rank_id][0], col_hi=blocks[rank_id][1])
        got = []

        def fetch_result(_k, _r, eng):            # on the rank that ran the inflation: result to the host, clusters
            fin = eng.result()
            interpret_result(fin)
            got.append(fin.nnz * 8 + (n + 1) * 8)

        stats = sharded_mcl_sweep(mc, inflations, a.max_iter, a.pruning, blocks, on_result=fetch_result)
        n_it = sum(st["rounds"] for st in stats)
        barrier()
        t2 = time.perf_counter()
        if s >= e2e_warm:
            e2e_t.append((t1 - t0, t2 - t1, n_it))
            d2h += sum(got)
            if rank_id == 0:
                d2h += sum(v.nbytes for v in table.values()) + tot.nbytes
        mc.close()
        mat.close()
        tab.close()
    d2h_all = torch.tensor([float(d2h)], dtype=torch.float64, device=dev)
    dist.all_reduce(d2h_all)                                # results are fetched by the rank that ran the inflation
    d2h = int(d2h_all.item())
    if rank_id == 0:
        build_ms = sum(s["build_ms"] for s in steps) / len(steps)
        mcl_ms = sum(s["mcl_ms"] for s in steps) / len(steps)
        e2e = None
        mcl_e2e = None
        if e2e_t:
            e2e = {"value": a.pairs / float(np.median([x[0] for x in e2e_t])), "unit": "pairs/s", "passes": len(e2e_t),
                   "h2d_bytes_per_step": 16 * a.pairs + 13 * n * world, "d2h_bytes_per_step": int(d2h / len(e2e_t))}
            mcl_e2e = {"value": sum(x[2] for x in e2e_t) / sum(x[1] for x in e2e_t), "unit": "iter/s"}
        line = {
            "metric": "hic_pairs_per_sec_matrix_build", "value": a.pairs / (build_ms / 1000.0), "unit": "pairs/s",
            "n_gpus": world, "steps": a.steps, "warmup": a.warmup, "ms_per_step": 1000.0 * wall / a.steps,
            "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "int32 counts / fp32 matrix",
            "data": "synthetic",
            "config": {"workload": B.workload_name(a), "inflations": inflations, "max_iter": a.max_iter,
                       "pruning": a.pruning, "parallelism": "pair stream sharded x{0}, records routed to the owner of their contig pair "
                       "(all-to-all), disjoint partition tables all-gathered; MCL: pre-expansion and iteration 0 of every inflation on "
                       "column blocks x{0}, one all-gather of pruned columns per inflation, then inflation k runs on rank k mod {0} "
                       "alone".format(world),
                       "cache": "inputs and the dense pre-expanded matrix exceed the 50 MB L2",
                       "step": "route + all-to-all + link build + partition all-gather + index + CSC + normalise + pre-expansion + "
                               "MCL sweep"},
            "stage_ms": {"link_build_and_matrix": build_ms, "mcl_sweep": mcl_ms},
            "mcl": {"metric": "mcl_iterations_per_sec", "value": steps[-1]["iters"] / (mcl_ms / 1000.0), "unit": "iter/s",
                    "iterations": steps[-1]["iters"], "e2e": mcl_e2e},
            "links": {"pairs": a.pairs, "nnz_full": steps[-1]["nnz_full"], "n_matrix": steps[-1]["n_matrix"]},
            "e2e": e2e, "gpu_launches": int(launches), "clocks": clocks,
            "roofline": rank0_roofline(steps[-1]),
            "cpu_baseline": None if a.no_cpu_baseline else B.cpu_baseline_block(a, asm, rank, in_nx, rec),
        }
        print(json.dumps(line))
    ctx.close()
    dist.destroy_process_group()
