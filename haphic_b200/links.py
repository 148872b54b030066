"""Host side of the link-counting path (hh_links / hh_matrix handles).

Mirrors the data the reference's ``parse_alignments_for_ctgs``
(scripts/HapHiC_cluster.py:1596-1655) and ``dict_to_matrix`` (310-373) produce, with the
per-read-pair loop running on the GPU.
"""

from __future__ import annotations

import ctypes as C
from collections import defaultdict

import numpy as np

from . import _lib
from ._lib import Context, LinksInfo, check, load, ptr

NONE32 = 0xFFFFFFFF

_PINNED = {}


def _host_buffer(tag, shape, dtype):
    """numpy array for D2H results.  Backed by page-locked memory (cached per tag and size, because
    cudaHostAlloc of gigabytes costs more than the copy) when torch is importable: pageable targets
    limit cudaMemcpy to a fraction of the PCIe rate."""
    n = int(np.prod(shape))
    if n * np.dtype(dtype).itemsize < (1 << 20):
        return np.empty(shape, dtype)
    try:
        import torch
        key = (tag, np.dtype(dtype).str)
        buf = _PINNED.get(key)
        nbytes = n * np.dtype(dtype).itemsize
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(int(nbytes * 1.25), dtype=torch.uint8, pin_memory=True)
            _PINNED[key] = buf
        return buf[:nbytes].numpy().view(dtype).reshape(shape)
    except Exception:
        return np.empty(shape, dtype)


def name_rank(names) -> np.ndarray:
    """Rank of every contig under Python ``str`` ordering of the names (the order
    ``sorted(((ref, pos+1), (mref, mpos+1)))`` uses, HapHiC_cluster.py:1629)."""
    order = sorted(range(len(names)), key=names.__getitem__)
    rank = np.empty(len(names), dtype=np.int32)
    rank[order] = np.arange(len(names), dtype=np.int32)
    return rank


class LinkTable:
    """Device-resident link counters of one run (full / flank / HT / per-fragment totals)."""
    _close_order = 0

    def __init__(self, ctx: Context, ctg_len, rank, in_nx, flank_bp: int, capacity_hint: int = 0, frags=None):
        """``frags`` switches to fragment mode (parse_alignments, 1658-1752): a dict with
        ``ctg_rank`` [n_src], ``frag_base`` [n_src+1] and ``bin_size``; then ctg_len / rank / in_nx describe
        the FRAGMENTS (contigs or bins) and every result of this table is in fragment ids."""
        self.ctx = ctx
        self.n_ctg = len(ctg_len)
        self._len = np.ascontiguousarray(ctg_len, dtype=np.int64)
        self._rank = np.ascontiguousarray(rank, dtype=np.int32)
        self._nx = np.ascontiguousarray(in_nx, dtype=np.uint8)
        if not (len(self._rank) == self.n_ctg == len(self._nx)):
            raise ValueError("ctg_len, rank and in_nx must have one entry per contig")
        self._h = C.c_void_p()
        if frags is None:
            check(load().hh_links_create(ctx.handle, self.n_ctg, ptr(self._len), ptr(self._rank), ptr(self._nx),
                                         int(flank_bp), int(capacity_hint), C.byref(self._h)))
        else:
            self._src_rank = np.ascontiguousarray(frags["ctg_rank"], dtype=np.int32)
            self._fbase = np.ascontiguousarray(frags["frag_base"], dtype=np.int32)
            check(load().hh_links_create_frags(ctx.handle, len(self._src_rank), ptr(self._src_rank), ptr(self._fbase),
                                               self.n_ctg, ptr(self._len), ptr(self._rank), ptr(self._nx),
                                               int(frags["bin_size"]), int(flank_bp), int(capacity_hint), C.byref(self._h)))
        ctx.adopt(self)
        self._stream_pos = 0
        self.info = None

    # -- streaming -------------------------------------------------------------------------
    def add(self, rec, stream_offset: int | None = None, asynchronous: bool = False):
        """Stream records: int32 [P, 4] (ctg_a, pos_a, ctg_b, pos_b); numpy array, pinned/pageable
        torch CPU tensor or torch CUDA tensor."""
        n_rec = int(rec.shape[0])
        if n_rec == 0:
            return
        off = self._stream_pos if stream_offset is None else int(stream_offset)
        if isinstance(rec, np.ndarray):
            if rec.dtype != np.int32 or rec.ndim != 2 or rec.shape[1] != 4 or not rec.flags.c_contiguous:
                rec = np.ascontiguousarray(rec, dtype=np.int32).reshape(-1, 4)
            mem = _lib.HH_MEM_HOST
        else:
            import torch
            if rec.dtype != torch.int32 or rec.dim() != 2 or rec.shape[1] != 4 or not rec.is_contiguous():
                raise ValueError("records must be a contiguous int32 [P, 4] tensor")
            mem = _lib.HH_MEM_DEVICE if rec.is_cuda else _lib.HH_MEM_HOST
            if rec.is_cuda:
                # the library works on its own (non-blocking) stream: whatever produced `rec` on torch's stream must be done
                torch.cuda.current_stream(rec.device).synchronize()
        if asynchronous:
            if mem != _lib.HH_MEM_DEVICE:
                raise ValueError("asynchronous add needs device-resident records")
            check(load().hh_links_add_async(self._h, ptr(rec), n_rec, off))
        else:
            check(load().hh_links_add(self._h, ptr(rec), n_rec, off, mem))
        self._stream_pos = max(self._stream_pos, off + n_rec)

    def finish(self) -> LinksInfo:
        info = LinksInfo()
        check(load().hh_links_finish(self._h, C.byref(info)))
        self.info = info
        return info

    def agg_info(self) -> dict:
        """How a partitioned count was aggregated at finish: hash buckets, those counted in shared memory, those counted
        by the global-table fallback (all 0 for a table counted directly)."""
        b, s, f = C.c_int64(), C.c_int64(), C.c_int64()
        check(load().hh_links_agg_info(self._h, C.byref(b), C.byref(s), C.byref(f)))
        return {"buckets": int(b.value), "smem_buckets": int(s.value), "fallback_buckets": int(f.value)}

    def record_bytes(self) -> dict:
        """Bytes per record of a partitioned count: ``sets``, one entry per partition set opened by the add calls, and
        ``buckets``, the bucket buffer of the finish (0 before it).  8 is the narrow format (at most 65,536 contigs and
        stream indices below 2^29), 16 the wide one; no sets and 0 for a table counted directly."""
        n, b = C.c_int32(), C.c_int32()
        check(load().hh_links_record_bytes(self._h, None, 0, C.byref(n), C.byref(b)))
        sets = (C.c_int32 * max(1, n.value))()
        check(load().hh_links_record_bytes(self._h, sets, n.value, C.byref(n), C.byref(b)))
        return {"sets": [int(x) for x in sets[:n.value]], "buckets": int(b.value)}

    # -- results ---------------------------------------------------------------------------
    def fetch(self, pinned: bool = False) -> dict:
        """Arrays of nnz_full entries in full_link_dict insertion order.  ``pinned=True`` returns views of
        cached page-locked buffers (full PCIe rate) that the next pinned fetch overwrites."""
        if self.info is None:
            self.finish()
        nnz = int(self.info.nnz_full)
        hb = _host_buffer if pinned else (lambda _tag, shape, dtype: np.empty(shape, dtype))
        out = {
            "key_i": hb("key_i", (nnz,), np.int32), "key_j": hb("key_j", (nnz,), np.int32),
            "full": hb("full", (nnz,), np.uint32), "flank": hb("flank", (nnz,), np.uint32),
            "first_full": hb("first_full", (nnz,), np.uint32), "first_flank": hb("first_flank", (nnz,), np.uint32),
            "ht": hb("ht", (nnz, 4), np.uint32),
        }
        check(load().hh_links_fetch(self._h, ptr(out["key_i"]), ptr(out["key_j"]), ptr(out["full"]), ptr(out["flank"]),
                                    ptr(out["first_full"]), ptr(out["first_flank"]), ptr(out["ht"])))
        return out

    def fetch_phased(self, hap, phasing_weight: float) -> dict:
        """full_link_dict after reduce_inter_hap_HiC_links (695-707) with ``hap`` (haplotype index per contig), reduced on the
        device (hh_links_fetch_phased): key_i, key_j, fp64 values and is_float (uint8) of the entries that remain, in dict
        insertion order."""
        if self.info is None:
            self.finish()
        hap = self._hap(hap)
        nnz = int(self.info.nnz_full)
        out = {"key_i": np.empty(nnz, np.int32), "key_j": np.empty(nnz, np.int32), "values": np.empty(nnz, np.float64),
               "is_float": np.empty(nnz, np.uint8)}
        n = C.c_int64()
        check(load().hh_links_fetch_phased(self._h, ptr(hap), float(phasing_weight), ptr(out["key_i"]), ptr(out["key_j"]),
                                           ptr(out["values"]), ptr(out["is_float"]), C.byref(n)))
        return {k: v[:int(n.value)] for k, v in out.items()}

    def fetch_ctg(self) -> np.ndarray:
        tot = np.empty(self.n_ctg, np.int64)
        check(load().hh_links_fetch_ctg(self._h, ptr(tot)))
        return tot

    def _hap(self, hap):
        if hap is None:
            return None
        hap = np.ascontiguousarray(hap, dtype=np.int32)
        if hap.shape != (self.n_ctg,):
            raise ValueError("hap must have one entry per fragment of the table")
        return hap

    def linked_index(self, keep, hap=None, phasing_weight: float = 0.0, normalize_by_nlinks: bool = False):
        """(index, n_linked): first-seen matrix index of every fragment present in
        flank_link_dict restricted to ``keep`` (HapHiC_cluster.py:327-349); -1 elsewhere.  With ``hap`` (haplotype index
        per fragment) the dict is the one reduce_inter_hap_HiC_links (695-707) leaves for ``phasing_weight``."""
        if self.info is None:
            self.finish()
        keep = np.ascontiguousarray(keep, dtype=np.uint8)
        hap = self._hap(hap)
        index = np.empty(self.n_ctg, np.int32)
        n_linked = C.c_int32()
        check(load().hh_links_linked_index_phased(self._h, ptr(keep), int(bool(normalize_by_nlinks)),
                                                  ptr(hap) if hap is not None else None, float(phasing_weight), ptr(index),
                                                  C.byref(n_linked)))
        return index, int(n_linked.value)

    def to_matrix(self, keep, tail=None, normalize_by_nlinks: bool = False, add_self_loops: bool = True, hap=None,
                  phasing_weight: float = 0.0, ul=None) -> "LinkMatrix":
        """dict_to_matrix on the device; ``hap`` / ``phasing_weight`` as in linked_index.  ``ul`` = (ul_path, ul_parent) per
        fragment doubles the flank links between two different contigs of one ultra-long-read path
        (hh_matrix_from_links_ex); the first-seen indices do not depend on it."""
        if self.info is None:
            self.finish()
        keep = np.ascontiguousarray(keep, dtype=np.uint8)
        tail = np.ascontiguousarray(tail if tail is not None else [], dtype=np.int32)
        hap = self._hap(hap)
        ul_path = ul_parent = None
        if ul is not None:
            ul_path, ul_parent = (np.ascontiguousarray(a, dtype=np.int32) for a in ul)
            if ul_path.shape != (self.n_ctg,) or ul_parent.shape != (self.n_ctg,):
                raise ValueError("ul_path and ul_parent must have one entry per fragment of the table")
        h = C.c_void_p()
        check(load().hh_matrix_from_links_ex(self._h, ptr(keep), ptr(tail) if len(tail) else None, len(tail),
                                             int(bool(normalize_by_nlinks)), int(bool(add_self_loops)),
                                             ptr(hap) if hap is not None else None, float(phasing_weight),
                                             ptr(ul_path) if ul is not None else None, ptr(ul_parent) if ul is not None else None,
                                             C.byref(h)))
        return LinkMatrix(self.ctx, h)

    def set_ul_pairs(self, key_i, key_j, ht_slot):
        """Contig pairs joined by ultra-long reads (hh_links_set_ul_pairs): fetch and fetch_phased then return their full
        count, and fetch their HT slot ``ht_slot`` (2 * ti + tj), doubled."""
        ki, kj, hs = (np.ascontiguousarray(a, dtype=np.int32) for a in (key_i, key_j, ht_slot))
        n = len(ki)
        if not (len(kj) == len(hs) == n):
            raise ValueError("key_i, key_j and ht_slot must have the same length")
        check(load().hh_links_set_ul_pairs(self._h, ptr(ki) if n else None, ptr(kj) if n else None, ptr(hs) if n else None, n))

    # -- multi-GPU -------------------------------------------------------------------------
    def export(self):
        """(entries [nnz, 9] uint32 CUDA tensor, ctg totals [n_ctg] int64 CUDA tensor, n_records, n_used)."""
        import torch
        if self.info is None:
            self.finish()
        dev = torch.device("cuda", self.ctx.device)
        ent = torch.empty((int(self.info.nnz_full), 9), dtype=torch.int32, device=dev)
        tot = torch.empty(self.n_ctg, dtype=torch.int64, device=dev)
        check(load().hh_links_export(self._h, ptr(ent), ptr(tot)))
        return ent, tot, int(self.info.n_records), int(self.info.n_used)

    def merge(self, entries, ctg_totals, n_records: int, n_used: int):
        n = int(entries.shape[0])
        check(load().hh_links_merge(self._h, ptr(entries) if n else None, n, ptr(ctg_totals), int(n_records), int(n_used)))
        self.info = None        # re-opened: finish() again

    # routed counting: route -> (all-to-all) -> add_routed -> finish_partition -> export -> (all-gather) -> adopt
    def route(self, rec, stream_offset: int, world: int):
        """Split a CUDA shard of the stream by owner rank.  Returns (records [m, 4] int32, stream indices [m] int32
        holding uint32 values, counts list of `world` ints); group d is rows sum(counts[:d]) .. sum(counts[:d+1])."""
        import torch
        if not rec.is_cuda or rec.dtype != torch.int32 or rec.dim() != 2 or rec.shape[1] != 4 or not rec.is_contiguous():
            raise ValueError("records must be a contiguous int32 [P, 4] CUDA tensor")
        n_rec = int(rec.shape[0])
        rec_out = torch.empty((max(n_rec, 1), 4), dtype=torch.int32, device=rec.device)
        pos_out = torch.empty(max(n_rec, 1), dtype=torch.int32, device=rec.device)
        counts = np.zeros(world, np.int64)
        check(load().hh_links_route(self._h, ptr(rec) if n_rec else None, n_rec, int(stream_offset), int(world),
                                    ptr(rec_out), ptr(pos_out), ptr(counts)))
        m = int(counts.sum())
        self._stream_pos = max(self._stream_pos, int(stream_offset) + n_rec)
        return rec_out[:m], pos_out[:m], [int(c) for c in counts]

    def add_routed(self, rec, pos):
        n_rec = int(rec.shape[0])
        if n_rec:
            check(load().hh_links_add_routed(self._h, ptr(rec), ptr(pos), n_rec))

    def finish_partition(self) -> LinksInfo:
        info = LinksInfo()
        check(load().hh_links_finish_partition(self._h, C.byref(info)))
        self.info = info
        return info

    def adopt(self, entries, ctg_totals, n_records: int, n_used: int, stream_end: int):
        n = int(entries.shape[0])
        check(load().hh_links_adopt(self._h, ptr(entries) if n else None, n, ptr(ctg_totals), int(n_records), int(n_used),
                                    int(stream_end)))
        self.info = None
        return self.finish()

    def close(self):
        if self._h:
            load().hh_links_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LinkMatrix:
    """The contig x contig link matrix on the device (hh_matrix): symmetric fp32, self loops = 1."""

    _close_order = 1

    def __init__(self, ctx: Context, handle):
        self.ctx = ctx
        self._h = handle
        ctx.adopt(self)
        n = C.c_int32()
        nnz = C.c_int64()
        check(load().hh_matrix_info(self._h, C.byref(n), C.byref(nnz)))
        self.n, self.nnz = int(n.value), int(nnz.value)

    @classmethod
    def from_csc(cls, ctx: Context, matrix) -> "LinkMatrix":
        """From a scipy CSC / anything ``scipy.sparse.csc_matrix`` accepts (host)."""
        import scipy.sparse as sp
        m = sp.csc_matrix(matrix, dtype=np.float32)
        if m.shape[0] != m.shape[1]:
            raise ValueError("link matrix must be square")
        indptr = np.ascontiguousarray(m.indptr, dtype=np.int64)
        indices = np.ascontiguousarray(m.indices, dtype=np.int32)
        data = np.ascontiguousarray(m.data, dtype=np.float32)
        h = C.c_void_p()
        check(load().hh_matrix_from_csc(ctx.handle, m.shape[0], ptr(indptr), ptr(indices), ptr(data), C.byref(h)))
        return cls(ctx, h)

    def rank_sums(self, topN: int = 10) -> np.ndarray:
        """rank-sum statistic of filter_fragments (864-892) per matrix index (matrix built without self loops)."""
        out = np.empty(self.n, np.int64)
        check(load().hh_matrix_rank_sums(self._h, int(topN), ptr(out)))
        return out

    def to_scipy(self):
        """Canonical (row-sorted, duplicates summed) CSC on the host."""
        import scipy.sparse as sp
        indptr = np.empty(self.n + 1, np.int64)
        check(load().hh_matrix_fetch_csc(self._h, ptr(indptr), None, None))
        nnz = int(indptr[-1])
        indices = np.empty(nnz, np.int32)
        data = np.empty(nnz, np.float32)
        check(load().hh_matrix_fetch_csc(self._h, ptr(indptr), ptr(indices), ptr(data)))
        return sp.csc_matrix((data, indices, indptr), shape=(self.n, self.n))

    def close(self):
        if self._h:
            load().hh_matrix_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GroupLinkStats:
    """The full links, resident on the device for the reassignment statistics of every inflation (hh_stats):
    parse_link_dict's (contig, group) sums, their ranking and the best-group statistics of output_statistics.  Any form of
    full_link_dict: integer counts (``is_float`` None), or ints and Python floats (``is_float`` per entry)."""

    _close_order = 1

    def __init__(self, ctx: Context, n_ctg: int, key_i, key_j, values, is_float=None):
        self.ctx = ctx
        self.n_ctg = int(n_ctg)
        ki = np.ascontiguousarray(key_i, dtype=np.int32)
        kj = np.ascontiguousarray(key_j, dtype=np.int32)
        v = np.ascontiguousarray(values, dtype=np.float64)
        m = len(ki)
        f = np.zeros(m, np.uint8) if is_float is None else np.ascontiguousarray(is_float, dtype=np.uint8)
        self._h = C.c_void_p()
        check(load().hh_stats_create(ctx.handle, self.n_ctg, ptr(ki) if m else None, ptr(kj) if m else None, ptr(v) if m else None,
                                     ptr(f) if m else None, m, C.byref(self._h)))
        ctx.adopt(self)
        self.n_ranked = 0

    def rank(self, group, n_groups: int) -> int:
        """Rank every contig's groups (``group`` per contig, -1 = ungrouped, else < n_groups); returns the number of sums."""
        g = np.ascontiguousarray(group, dtype=np.int32)
        if g.shape != (self.n_ctg,):
            raise ValueError("group must have one entry per contig")
        n = C.c_int64()
        check(load().hh_stats_rank(self._h, ptr(g), int(n_groups), C.byref(n)))
        self.n_ranked = int(n.value)
        return self.n_ranked

    def fetch_ranked(self):
        """(contig, group, links, is_float) of the last ranking, ordered by (contig, rank)."""
        n = self.n_ranked
        c, g = np.empty(n, np.int32), np.empty(n, np.int32)
        s, f = np.empty(n, np.float64), np.empty(n, np.uint8)
        check(load().hh_stats_fetch_ranked(self._h, ptr(c), ptr(g), ptr(s), ptr(f)))
        return c, g, s, f.astype(bool)

    def best(self, group_re, ctg_re, compensated: bool) -> dict:
        """Per contig over the last ranking: has, top_links, top_is_float, top_density, others, ratio (hh_stats_best)."""
        gre = np.ascontiguousarray(group_re, dtype=np.int64)
        cre = np.ascontiguousarray(ctg_re, dtype=np.int64)
        if cre.shape != (self.n_ctg,):
            raise ValueError("ctg_re must have one entry per contig")
        n = self.n_ctg
        out = {"has": np.empty(n, np.uint8), "top_links": np.empty(n, np.float64), "top_is_float": np.empty(n, np.uint8),
               "top_density": np.empty(n, np.float64), "others": np.empty(n, np.float64), "ratio": np.empty(n, np.float64)}
        check(load().hh_stats_best(self._h, ptr(gre), len(gre), ptr(cre), int(bool(compensated)), ptr(out["has"]),
                                   ptr(out["top_links"]), ptr(out["top_is_float"]), ptr(out["top_density"]), ptr(out["others"]),
                                   ptr(out["ratio"])))
        return out

    def close(self):
        if self._h:
            load().hh_stats_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------
# reference-shaped view of a finished LinkTable
# ------------------------------------------------------------------------------------------

def link_dicts(table: LinkTable, names):
    """(full_link_dict, flank_link_dict, HT_link_dict, ctg_link_dict) as the reference builds them
    (HapHiC_cluster.py:1605-1649): ``defaultdict(int)`` keyed by name tuples, in insertion order."""
    f = table.fetch()
    ki, kj = f["key_i"].tolist(), f["key_j"].tolist()
    full_link_dict = defaultdict(int)
    for a, b, v in zip(ki, kj, f["full"].tolist()):
        full_link_dict[(names[a], names[b])] = v
    # flank_link_dict is ordered by the first flank-qualifying record of each pair
    sel = np.nonzero(f["flank"] > 0)[0]
    sel = sel[np.argsort(f["first_flank"][sel], kind="stable")]
    flank_link_dict = defaultdict(int)
    for e in sel.tolist():
        flank_link_dict[(names[ki[e]], names[kj[e]])] = int(f["flank"][e])
    # HT_link_dict keys appear when their first record does; within the 4-way split of one pair the
    # order is not recoverable from counters alone, so entries are grouped by pair (consumers look
    # keys up, HapHiC_sort.py:126-131, and never iterate in order)
    HT_link_dict = defaultdict(int)
    suffix = ("_H", "_T")
    ht = f["ht"]
    for e, (a, b) in enumerate(zip(ki, kj)):
        for c in range(4):
            v = int(ht[e, c])
            if v:
                HT_link_dict[(names[a] + suffix[c >> 1], names[b] + suffix[c & 1])] = v
    tot = table.fetch_ctg()
    ctg_link_dict = defaultdict(int)
    # insertion order = first touch (i before j) over flank-qualifying records
    touch = {}
    for e in sel.tolist():
        t = int(f["first_flank"][e]) * 2
        a, b = ki[e], kj[e]
        if t < touch.get(a, 1 << 62):
            touch[a] = t
        if t + 1 < touch.get(b, 1 << 62):
            touch[b] = t + 1
    for c in sorted(touch, key=touch.__getitem__):
        ctg_link_dict[names[c]] = int(tot[c])
    return full_link_dict, flank_link_dict, HT_link_dict, ctg_link_dict
