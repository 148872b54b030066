"""`haphic plot` on the GPU: a drop-in for scripts/HapHiC_plot.py (v1.0.7).

The AGP layout and the per-(contig, aln bin) candidate ranges are built here on the host (parse_agp 41-103,
generate_contact_matrix 106-150).  Records come from the native .pairs / BAM readers (hicio) and are binned on the device
(hh_contact_*, csrc/hh_plot.cu), which also symmetrises the matrix, balances it with Knight-Ruiz and produces the
normalised matrix and its vmax median.  Drawing is matplotlib's, imported only when a figure is drawn.

    python -m haphic_b200.plot asm.agp aln.pairs [options]
"""

from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import logging
import os
import pickle
import sys
import time
from collections import OrderedDict, defaultdict
from math import ceil

import numpy as np

from . import _lib
from ._lib import Context, check, load, ptr

__version__ = "1.0.7-b200.1"
__update_time__ = "2026.09.24"

logging.basicConfig(format="%(asctime)s <%(filename)s> [%(funcName)s] %(message)s", datefmt="%Y-%m-%d %H:%M:%S")
logger = logging.getLogger(__name__)
logger.setLevel(logging.INFO)

CONVERGE_MSG = ("Unable to converge. Maybe the matrix is too sparse (too few Hi-C links). "
                "You can try another normalization method.")
NORM_MODE = {"KR": 0, "log10": 1, "none": 2}
SKIP, MISSING = -1, -2


# ------------------------------------------------------------------------------------------------
# AGP layout (host)
# ------------------------------------------------------------------------------------------------

class Layout:
    """What parse_agp and generate_contact_matrix produce, as arrays the device can use.

    ``names``: contigs with a W line, in order of first appearance (the record ids);  ``group_size``: scaffold -> end of
    its last W line;  ``group_list`` / ``nb``: kept scaffolds and total bins;  ``in_set``: per contig, in ctg_set;
    ``slot_base`` / ``cand_off`` / ``cand_lo`` / ``cand_hi`` / ``cand_bin``: ctg_aln_dict flattened, each range with the
    total bin of its (last) ctg_dict mapping, -1 when its scaffold is not kept, -2 when the scaffold has no such bin."""

    def __init__(self, agp, bin_size, min_len=1, specified_scaffolds=None):
        self.bin_size = int(bin_size)
        lines = []              # (group, group_start, group_end, ctg, raw_start, raw_end, ori)
        group_size = OrderedDict()
        with open(agp) as f:
            for line in f:
                if line.startswith("#") or not line.strip():
                    continue
                cols = line.split()
                if cols[4] != "W":
                    continue
                gs, ge, rs, re_ = int(cols[1]), int(cols[2]), int(cols[6]), int(cols[7])
                group_size[cols[0]] = ge
                lines.append((cols[0], gs, ge, cols[5], rs, re_, cols[8]))
        self.group_size = group_size
        bs = self.bin_size

        # kept scaffolds and their bins (generate_contact_matrix)
        if specified_scaffolds:
            order = specified_scaffolds.split(",")
            for g in order:
                if g not in group_size:
                    raise RuntimeError("Cannot find {} in the input AGP file".format(g))
        else:
            order = [g for g, s in group_size.items() if s >= min_len * 1000000]
        self.group_list = list(order)
        total = dict()
        nb = 0
        for g in order:
            nbins = group_size[g] // bs + 1
            for k in range(nbins):
                total[(g, k)] = nb + k
            nb += nbins
        self.nb = nb
        kept = set(order)

        names = []
        ctg_id = {}
        for ln in lines:
            if ln[3] not in ctg_id:
                ctg_id[ln[3]] = len(names)
                names.append(ln[3])
        self.names = names
        # ctg_set: contigs of the fragments (contig, raw start, raw end) left after those of every dropped scaffold are
        # removed -- a fragment also placed in a kept scaffold goes too
        frags = {(ln[3], ln[4], ln[5]) for ln in lines}
        if not specified_scaffolds:
            frags -= {(ln[3], ln[4], ln[5]) for ln in lines if ln[0] not in kept}
        in_set = np.zeros(len(names), np.uint8)
        for ctg, _rs, _re in frags:
            in_set[ctg_id[ctg]] = 1
        self.in_set = in_set

        # ctg_dict (last mapping of a range wins) and ctg_aln_dict (every range, listed per aln bin it touches)
        mapping = defaultdict(dict)
        aln = defaultdict(lambda: defaultdict(list))
        for g, gs, ge, ctg, rs, re_, ori in lines:
            for gb in range((gs - 1) // bs, (ge - 1) // bs + 1):
                lo, hi = max(gb * bs + 1, gs), min((gb + 1) * bs, ge)
                if ori == "+":
                    a, b = lo - gs + rs, hi - gs + rs
                else:
                    assert ori == "-"
                    a, b = re_ - (hi - gs), re_ - (lo - gs)
                mapping[ctg][(a, b)] = (g, gb)
                for ab in range((a - 1) // bs, (b - 1) // bs + 1):
                    aln[ctg][ab].append((a, b))
        slot_base = np.zeros(len(names) + 1, np.int64)
        offs, lo_l, hi_l, bin_l = [0], [], [], []
        for c, ctg in enumerate(names):
            bins = aln[ctg]
            n_slot = max(bins) + 1 if bins else 0
            slot_base[c + 1] = slot_base[c] + n_slot
            for ab in range(n_slot):
                for rng in bins.get(ab, ()):
                    g, gb = mapping[ctg][rng]
                    lo_l.append(rng[0])
                    hi_l.append(rng[1])
                    bin_l.append(total.get((g, gb), MISSING) if g in kept else SKIP)
                offs.append(len(lo_l))
        self.slot_base = slot_base
        self.cand_off = np.asarray(offs, np.int64)
        self.cand_lo = np.asarray(lo_l, np.int64)
        self.cand_hi = np.asarray(hi_l, np.int64)
        self.cand_bin = np.asarray(bin_l, np.int32)

    def name_index(self):
        from .hicio import NameIndex
        return NameIndex(self.names)

    def resolve(self, ctg, pos):
        """convert_group_bin_id on the host tables: the total bin, None (skip) or MISSING (the reference raises)."""
        c = self.name_index()[ctg]
        ab = (pos - 1) // self.bin_size
        s0, s1 = self.slot_base[c], self.slot_base[c + 1]
        if ab < 0 or ab >= s1 - s0 or self.cand_off[s0 + ab] == self.cand_off[s0 + ab + 1]:
            return MISSING
        for k in range(self.cand_off[s0 + ab], self.cand_off[s0 + ab + 1]):
            if self.cand_lo[k] <= pos <= self.cand_hi[k]:
                b = int(self.cand_bin[k])
                return None if b == SKIP else b
        return None

    def blocks(self):
        """(offset, bins) of every kept scaffold as normalize_matrix places them: ceil(size / bin_size) bins each."""
        out, start = [], 0
        for g in self.group_list:
            n = ceil(self.group_size[g] / self.bin_size)
            out.append((start, n))
            start += n
        return out


# ------------------------------------------------------------------------------------------------
# device handle
# ------------------------------------------------------------------------------------------------

def _records(rec):
    if isinstance(rec, np.ndarray):
        return np.ascontiguousarray(rec, dtype=np.int32).reshape(-1, 4), _lib.HH_MEM_HOST
    import torch
    if rec.dtype != torch.int32 or rec.dim() != 2 or rec.shape[1] != 4 or not rec.is_contiguous():
        raise ValueError("records must be a contiguous int32 [P, 4] tensor")
    if rec.is_cuda:
        # the library works on its own (non-blocking) stream: whatever produced `rec` on torch's stream must be done
        torch.cuda.current_stream(rec.device).synchronize()
        return rec, _lib.HH_MEM_DEVICE
    return rec, _lib.HH_MEM_HOST


def available_bytes(ctx) -> int:
    b = C.c_size_t()
    check(load().hh_ctx_mem_available(ctx.handle, C.byref(b)))
    return int(b.value)


def check_footprint(ctx, nb, count_bytes=4, blocks=(), figure=True):
    """Raise MemoryError unless the count matrix, the sorted intra-scaffold values of the vmax median and, when a figure is
    drawn, a 256 MB output staging block fit the device."""
    n_val = sum(n * (n - 1) for _o, n in blocks)
    need = nb * nb * count_bytes + 2 * 8 * n_val + (256 << 20 if figure else 0)
    have = available_bytes(ctx)
    if need > have:
        raise MemoryError("the {}-bin contact map needs {} bytes of device memory ({} bytes of counts); {} bytes are "
                          "available".format(nb, need, nb * nb * count_bytes, have))


class ContactMap:
    """The device contact matrix of one run: counting, the symmetrised int64 matrix, KR and normalisation."""
    _close_order = 0

    def __init__(self, ctx: Context, layout: Layout = None, counts=None):
        """From a layout (counting records), or from a symmetrised int64 matrix ``counts`` (a contact_matrix.pkl)."""
        self.ctx = ctx
        self._h = C.c_void_p()
        self.layout = layout
        if counts is not None:
            self._counts = np.ascontiguousarray(counts, dtype=np.int64)
            self.nb = int(self._counts.shape[0])
            check(load().hh_contact_load(ctx.handle, self.nb, ptr(self._counts), C.byref(self._h)))
            self.finished = True
        else:
            L = layout
            self.nb = L.nb
            check(load().hh_contact_create(ctx.handle, len(L.names), ptr(L.in_set), ptr(L.slot_base), ptr(L.cand_off),
                                           ptr(L.cand_lo), ptr(L.cand_hi), ptr(L.cand_bin), L.nb, L.bin_size,
                                           C.byref(self._h)))
            self.finished = False
        ctx.adopt(self)

    def add(self, rec, asynchronous=False):
        """Count records int32 [P, 4] (id_a, pos_a, id_b, pos_b; 0-based positions) in stream order: a numpy array, a
        torch CPU tensor or a torch CUDA tensor; ``asynchronous`` (device records) returns before they are counted."""
        rec, mem = _records(rec)
        n = int(rec.shape[0])
        if n == 0:
            return
        if asynchronous:
            if mem != _lib.HH_MEM_DEVICE:
                raise ValueError("asynchronous add needs device-resident records")
            check(load().hh_contact_add_async(self._h, ptr(rec), n))
        else:
            check(load().hh_contact_add(self._h, ptr(rec), n, mem))

    def error(self):
        """(stream index, end, contig id, 1-based position) of the first record the AGP cannot place, or None."""
        idx, end, ctg, pos = C.c_int64(), C.c_int32(), C.c_int32(), C.c_int64()
        check(load().hh_contact_error(self._h, C.byref(idx), C.byref(end), C.byref(ctg), C.byref(pos)))
        if idx.value < 0:
            return None
        return int(idx.value), int(end.value), int(ctg.value), int(pos.value)

    def finish(self):
        check(load().hh_contact_finish(self._h))
        self.finished = True

    @property
    def count_bytes(self):
        b = C.c_int32()
        check(load().hh_contact_info(self._h, None, C.byref(b), None))
        return int(b.value)

    def fetch(self) -> np.ndarray:
        out = np.empty((self.nb, self.nb), np.int64)
        check(load().hh_contact_fetch(self._h, ptr(out)))
        return out

    def kr(self, blocks, tol=1e-6, delta=0.1, Delta=3, max_outer=1000, max_inner=10000):
        """bnewt on every block (offset, bins) of counts + 1e-5, advanced together.  Returns [(x, outer steps, inner
        steps, converged)] per block."""
        off = np.ascontiguousarray([b[0] for b in blocks], np.int32)
        n = np.ascontiguousarray([b[1] for b in blocks], np.int32)
        x = np.empty(int(n.sum()), np.float64)
        n_outer = np.zeros(len(blocks), np.int32)
        n_inner = np.zeros(len(blocks), np.int64)
        status = np.zeros(len(blocks), np.int32)
        check(load().hh_contact_kr(self._h, len(blocks), ptr(off), ptr(n), float(tol), float(delta), float(Delta),
                                   int(max_outer), int(max_inner), ptr(x), ptr(n_outer), ptr(n_inner), ptr(status)))
        res, s = [], 0
        for q in range(len(blocks)):
            res.append((x[s:s + n[q]].copy(), int(n_outer[q]), int(n_inner[q]), status[q] == 0))
            s += int(n[q])
        return res

    def normalize(self, mode, blocks, x_blocks=None, x_whole=None, want_matrix=True):
        """(normalised nb x nb fp64 matrix or None, median of the off-diagonal block entries)."""
        off = np.ascontiguousarray([b[0] for b in blocks], np.int32)
        n = np.ascontiguousarray([b[1] for b in blocks], np.int32)
        xb = None if x_blocks is None else np.ascontiguousarray(x_blocks, np.float64)
        xw = None if x_whole is None else np.ascontiguousarray(x_whole, np.float64)
        out = np.empty((self.nb, self.nb), np.float64) if want_matrix else None
        lo, hi, nv = C.c_double(), C.c_double(), C.c_int64()
        check(load().hh_contact_normalize(self._h, NORM_MODE[mode], len(blocks), ptr(off), ptr(n), ptr(xb), ptr(xw), ptr(out),
                                          C.byref(lo), C.byref(hi), C.byref(nv)))
        if nv.value == 0:
            median = np.float64(np.nan)
        elif nv.value % 2:
            median = np.float64(lo.value)
        else:
            median = np.mean(np.array([lo.value, hi.value]))
        return out, median

    def close(self):
        if self._h:
            load().hh_contact_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def kr_balance(matrix, blocks=None, ctx=None, **kw):
    """bnewt (291-404) of ``matrix + 1e-5`` for a symmetrised int64 count matrix on the device: every (offset, bins) of
    ``blocks`` (default: the whole matrix) is balanced, all in the same launches.  Returns [(x, outer, inner, converged)]."""
    own = ctx is None
    ctx = Context(0) if own else ctx
    try:
        cm = ContactMap(ctx, counts=matrix)
        try:
            return cm.kr(blocks if blocks is not None else [(0, int(np.asarray(matrix).shape[0]))], **kw)
        finally:
            cm.close()
    finally:
        if own:
            ctx.close()


# ------------------------------------------------------------------------------------------------
# the run
# ------------------------------------------------------------------------------------------------

def get_file_md5(filename):
    with open(filename, "rb") as f:
        return hashlib.md5(f.read()).hexdigest()


def output_pickle(contact_matrix, args):
    logger.info("Writing raw contact matrix to a pickle file...")
    agp_md5 = get_file_md5(args.agp)
    with open("contact_matrix.pkl", "wb") as fpkl:
        pickle.dump((contact_matrix, args, agp_md5), fpkl)


def load_pickle(pickle_file, args):
    logger.info("Reading raw contact matrix from a previously generated pickle file...")
    with open(pickle_file, "rb") as fpkl:
        contact_matrix, old_args, agp_md5_pkl = pickle.load(fpkl)[:3]
    agp_md5_new = get_file_md5(args.agp)
    if agp_md5_pkl != agp_md5_new:
        msg = "The AGP file used to generate {} (md5: {}) is different from the input AGP file {} (md5: {})".format(
            pickle_file, agp_md5_pkl, args.agp, agp_md5_new)
        logger.error(msg)
        raise RuntimeError(msg)
    if (old_args.bin_size != args.bin_size or old_args.min_len != args.min_len
            or old_args.specified_scaffolds != args.specified_scaffolds):
        msg = ("The input parameters (--bin_size {} --min_len {} --specified_scaffolds {}) are not consistent with "
               "those used to generate `contact_map.pkl` (--bin_size {} --min_len {} --specified_scaffolds {})".format(
                   args.bin_size, args.min_len, args.specified_scaffolds,
                   old_args.bin_size, old_args.min_len, old_args.specified_scaffolds))
        logger.error(msg)
        raise RuntimeError(msg)
    return contact_matrix


def count_contacts(cm, layout, alignments, threads=8):
    """parse_pairs / parse_bam into the device matrix, raising the reference's error for the first unplaceable record."""
    from . import hicio
    names = layout.name_index()
    if alignments.endswith(".bam"):
        logger.info("Parsing input BAM file...")
        batches, what = hicio.bam_batches(alignments, names, inter_only=False, threads=threads), "BAM files"
    else:
        assert alignments.endswith(".pairs") or alignments.endswith(".pairs.gz")
        logger.info("Parsing input pairs file...")
        fmt = "pairs" if alignments.endswith(".pairs") else "bgzipped_pairs"
        batches, what = hicio.pairs_batches(alignments, fmt, names, bed_path=None, inter_only=False), ".pairs files"
    for rec in batches:
        cm.add(rec)
        if cm.error() is not None:
            break
    err = cm.error()
    if err is not None:
        _idx, _end, ctg, pos = err
        msg = ("Cannot find alignment position: {}:{} in the input AGP file. Please check whether the input AGP and {} "
               "match".format(layout.names[ctg], pos, what))
        logger.error(msg)
        raise Exception(msg)
    cm.finish()


def normalize_matrix(cm, layout, normalization, vmax_coef, manual_vmax, want_matrix=True, raw=None):
    """normalize_matrix (407-504) on the device: (normalised matrix or None, vmax)."""
    blocks = layout.blocks()
    if normalization == "KR":
        logger.info("Normalizing contact mattrix using the Knight-Ruiz (KR) balancing algorithm")
        res = cm.kr(blocks + [(0, cm.nb)])
        if not all(r[3] for r in res):
            logger.info(CONVERGE_MSG)
            raise RuntimeError(CONVERGE_MSG)
        xb = np.ones(cm.nb, np.float64)
        for (o, n), r in zip(blocks, res[:-1]):
            xb[o:o + n] = r[0]
        mat, median = cm.normalize("KR", blocks, xb, res[-1][0], want_matrix)
        if manual_vmax < 0:
            vmax = median * vmax_coef
            logger.info("The vmax for the KR-normalized matrix is calculated to be {} ({} * median)".format(vmax, vmax_coef))
        else:
            vmax = manual_vmax
            logger.info("The vmax for the KR-normalized matrix is manually designated as {})".format(vmax))
        return mat, vmax
    if normalization == "log10":
        logger.info("Normalizing contact matrix using log10...")
    else:
        logger.info("Normalization is disabled")
    mat, median = cm.normalize(normalization, blocks, want_matrix=want_matrix and normalization == "log10")
    if normalization == "none":
        mat = raw
    vmax = median * vmax_coef if manual_vmax < 0 else manual_vmax
    kind = "log-normalized" if normalization == "log10" else "raw"
    if manual_vmax < 0:
        logger.info("The vmax for the {} matrix is calculated to be {} ({} * median)".format(kind, vmax, vmax_coef))
    else:
        logger.info("The vmax for the {} matrix is manually designated as {}".format(kind, vmax))
    return mat, vmax


# ---- drawing (507-715), matplotlib imported lazily ------------------------------------------------

def _resolution(length, n):
    for r in (0.1, 0.25, 0.5, 1, 2.5, 5, 10, 25, 50, 100, 250, 500, 1000, 2500, 5000):
        if length // int(r * 1000000) + 1 < n:
            return r


def _xticks(length, resolution, bin_size):
    ticks, values = [], []
    for x in range(0, length + 1, int(resolution * 1000000)):
        ticks.append(x // bin_size)
        values.append(x / 1000000)
    if any(v != int(v) for v in values):
        return ticks, [str(v) for v in values]
    return ticks, [str(int(v)) for v in values]


def _set_origin(ax, n, origin):
    ax.axis({"bottom_left": [0, n, 0, n], "top_left": [0, n, n, 0], "bottom_right": [n, 0, 0, n]}.get(origin, [n, 0, n, 0]))


def _cmap(cmap):
    if "," in cmap:
        from matplotlib import colors
        return colors.LinearSegmentedColormap.from_list("my_cmap", cmap.split(","))
    return cmap


def _imshow(ax, m, cmap, vmax):
    from matplotlib import colors
    hm = ax.imshow(m, cmap=cmap)
    hm.set_norm(colors.Normalize(vmin=0, vmax=vmax))
    return hm


def _line_style(style):
    return (0, (10, 20)) if style == "dashed" else "solid"


def _out_file(args, stem):
    return "{}{}.{}".format(args.prefix or "", stem, args.output_format)


def draw_heatmap(plt, m, layout, vmax, args):
    logger.info("Drawing heatmap...")
    bs = layout.bin_size
    plt.rcParams["pdf.fonttype"] = 42
    fig, ax = plt.subplots(figsize=(args.figure_width / 2.54, args.figure_height / 2.54), dpi=1000)
    plt.subplots_adjust(bottom=0.05, left=0.15, right=1, top=0.95)
    ytick, yticks, edges = 0, [], []
    for g in layout.group_list:
        n = ceil(layout.group_size[g] / bs)
        yticks.append(ytick + n / 2)
        ytick += n
        edges.append(ytick - 0.5)
    ax.set_yticks(yticks)
    ax.set_yticklabels(layout.group_list, size=args.tick_label_size)
    nbins = m.shape[0]
    ticks, labels = _xticks(nbins * bs, _resolution(nbins * bs, 10), bs)
    ax.set_xticks(ticks)
    ax.set_xticklabels(labels, size=args.tick_label_size)
    _set_origin(ax, nbins, args.origin)
    hm = _imshow(ax, m, _cmap(args.cmap), vmax)
    ax.set_title("{} contact map (bin size: {} Kb, x-axis unit: Mb)".format(args.data_type, args.bin_size), fontsize=args.title_size)
    if args.border_style == "grid":
        ls = _line_style(args.gridline_style)
        for e in edges[:-1]:
            ax.vlines(e, 0, nbins, color=args.gridline_color, linestyle=ls, linewidth=args.gridline_width)
            ax.hlines(e, 0, nbins, color=args.gridline_color, linestyle=ls, linewidth=args.gridline_width)
    else:
        ls = _line_style(args.outline_style)
        last = 0
        for e in edges:
            for fn, a, b, c in ((ax.vlines, e, last, e), (ax.hlines, e, last, e), (ax.vlines, last, last, e), (ax.hlines, last, last, e)):
                fn(a, b, c, color=args.outline_color, linestyle=ls, linewidth=args.outline_width)
            last = e
    cb = fig.colorbar(hm, shrink=0.5)
    cb.set_label({"KR": "KR normalized counts", "log10": "Log$_{10}$(counts+1)"}.get(args.normalization, "Counts"),
                 fontsize=args.title_size)
    cb.ax.tick_params(labelsize=args.tick_label_size)
    plt.savefig(_out_file(args, "contact_map"), format=args.output_format)
    plt.close()


def draw_separate_heatmaps(plt, m, layout, vmax, args):
    logger.info("Drawing heatmap for each scaffold...")
    bs = layout.bin_size
    plt.rcParams["pdf.fonttype"] = 42
    groups = layout.group_list
    nrows = ceil(len(groups) / args.ncols)
    fig, axes = plt.subplots(nrows, args.ncols, figsize=(args.figure_width / 2.54,
                                                         ((args.figure_width - 2) * (nrows / args.ncols) * 1.2) / 2.54), dpi=1000)
    axs = []
    for n, ax in enumerate(np.asarray(axes).flat):
        if n < len(groups):
            axs.append(ax)
        elif len(groups) > args.ncols:
            fig.delaxes(axes[n // args.ncols, n % args.ncols])
        else:
            fig.delaxes(axes[n % args.ncols])
    start = 0
    for n, g in enumerate(groups):
        nbins = ceil(layout.group_size[g] / bs)
        gm = m[start:start + nbins, start:start + nbins]
        start += nbins
        ax = axs[n]
        k = gm.shape[0]
        ticks, labels = _xticks(k * bs, _resolution(k * bs, 6), bs)
        ax.set_xticks(ticks)
        ax.set_xticklabels(labels, size=args.tick_label_size_separate_plots)
        ax.set_yticks(ticks)
        ax.set_yticklabels(labels, size=args.tick_label_size_separate_plots)
        _set_origin(ax, k, args.origin)
        _imshow(ax, gm, _cmap(args.cmap), vmax)
        ax.set_title(g, fontsize=args.title_size_separate_plots)
    fig.tight_layout()
    plt.savefig(_out_file(args, "separate_plots"), format=args.output_format)
    plt.close()


def _pyplot():
    try:
        import matplotlib
        matplotlib.use("Agg")
        import matplotlib.pyplot as plt
        return plt
    except Exception:
        logger.warning("Module matplotlib is not correctly installed, HapHiC will NOT draw the contact maps")
        return None


def build_parser():
    p = argparse.ArgumentParser(prog="haphic plot")
    p.add_argument("agp", help="scaffolding result in AGP format. The IDs in this file should match those in the BAM file")
    p.add_argument("alignments", help="filtered Hi-C read alignments in BAM/pairs format or previously generated "
                                      "`contact_matrix.pkl` (much faster)")
    p.add_argument("--bin_size", type=int, default=500, help="bin size for generating contact matrix, default: %(default)s (kbp)")
    p.add_argument("--specified_scaffolds", default=None,
                   help="specify scaffolds to visualize, separated with commas, default: %(default)s. Disables --min_len")
    p.add_argument("--min_len", type=int, default=1, help="minimum scaffold length for visualization, default: %(default)s (Mbp)")
    p.add_argument("--data_type", default="Hi-C", help="data type in the heatmap title, default: %(default)s")
    p.add_argument("--cmap", default="white,red", help="colormap for the heatmap, default: %(default)s")
    p.add_argument("--normalization", choices=("KR", "log10", "none"), default="KR",
                   help="method for matrix normalization, default: %(default)s")
    p.add_argument("--vmax_coef", type=float, default=4.0,
                   help="values above vmax_coef times the median of the intra-scaffold matrices share one color, default: %(default)s")
    p.add_argument("--manual_vmax", type=float, default=-1, help="manually designate vmax, default: disabled")
    p.add_argument("--separate_plots", default=False, action="store_true",
                   help="generate `separate_plots.pdf` with one heatmap per scaffold, default: %(default)s")
    p.add_argument("--ncols", type=int, default=5, help="scaffolds per row in `separate_plots.pdf`, default: %(default)s")
    p.add_argument("--origin", choices=("bottom_left", "top_left", "bottom_right", "top_right"), default="bottom_left",
                   help="origin of each heatmap, default: %(default)s")
    p.add_argument("--border_style", choices=("grid", "outline"), default="grid", help="border style for scaffolds, default: %(default)s")
    p.add_argument("--gridline_color", default="grey", help="color for gridlines, default: %(default)s")
    p.add_argument("--gridline_style", choices=("solid", "dashed"), default="solid", help="style for gridlines, default: %(default)s")
    p.add_argument("--gridline_width", type=float, default=0.2, help="width for gridlines, default: %(default)s")
    p.add_argument("--outline_color", default="blue", help="color for outlines, default: %(default)s")
    p.add_argument("--outline_style", choices=("solid", "dashed"), default="solid", help="style for outlines, default: %(default)s")
    p.add_argument("--outline_width", type=float, default=0.2, help="width for outlines, default: %(default)s")
    p.add_argument("--figure_width", type=int, default=15, help="figure width, default: %(default)s (cm)")
    p.add_argument("--figure_height", type=int, default=12, help="figure height, default: %(default)s (cm)")
    p.add_argument("--output_format", choices={"pdf", "svg", "tiff", "png", "jpeg", "jpg"}, default="pdf",
                   help="output figure format, default: %(default)s")
    p.add_argument("--tick_label_size", type=int, default=6, help="tick label font size, default: %(default)s")
    p.add_argument("--title_size", type=int, default=7, help="title font size, default: %(default)s")
    p.add_argument("--tick_label_size_separate_plots", type=int, default=5,
                   help="tick label font size for separate plots, default: %(default)s")
    p.add_argument("--title_size_separate_plots", type=int, default=6, help="title font size for separate plots, default: %(default)s")
    p.add_argument("--prefix", default=None, help="prefix for output figure files, default: %(default)s")
    p.add_argument("--threads", type=int, default=8, help="number of threads for reading BAM file, default: %(default)s")
    return p


def parse_arguments(argv=None):
    return build_parser().parse_args(argv)


def run(args, log_file=None, ctx=None):
    """main() of the reference: contact_matrix.pkl (unless the alignments are one), the normalisation's log lines and the
    figures.  Returns (raw int64 matrix, normalised matrix, vmax)."""
    if log_file:
        handler = logging.FileHandler(log_file, "w")
        handler.setFormatter(logging.Formatter(fmt="%(asctime)s <%(filename)s> [%(funcName)s] %(message)s",
                                               datefmt="%Y-%m-%d %H:%M:%S"))
        logger.addHandler(handler)
    start_time = time.time()
    logger.info("Program started, HapHiC version: {} (update: {})".format(__version__, __update_time__))
    logger.info("Python version: {}".format(sys.version.replace("\n", "")))
    logger.info("Command: {}".format(" ".join(sys.argv)))
    bin_size = args.bin_size * 1000
    logger.info("Parsing input AGP file...")
    layout = Layout(args.agp, bin_size, args.min_len, args.specified_scaffolds)
    logger.info("Generating an empty contact matrix...")
    plt = _pyplot()
    own = ctx is None
    ctx = Context(0) if own else ctx
    try:
        if args.alignments.endswith(".pkl"):
            raw = load_pickle(args.alignments, args)
            check_footprint(ctx, raw.shape[0], 8 if raw.size and raw.max() > 2**31 - 1 else 4, layout.blocks(), plt is not None)
            cm = ContactMap(ctx, counts=raw)
        else:
            check_footprint(ctx, layout.nb, 4, layout.blocks(), plt is not None)
            cm = ContactMap(ctx, layout)
            count_contacts(cm, layout, args.alignments, args.threads)
            raw = cm.fetch()
            output_pickle(raw, args)
        try:
            norm, vmax = normalize_matrix(cm, layout, args.normalization, args.vmax_coef, args.manual_vmax,
                                          want_matrix=plt is not None, raw=raw)
        finally:
            cm.close()
    finally:
        if own:
            ctx.close()
    if plt is not None:
        draw_heatmap(plt, norm, layout, vmax, args)
        if args.separate_plots:
            draw_separate_heatmaps(plt, norm, layout, vmax, args)
    logger.info("Program finished in {}s".format(time.time() - start_time))
    return raw, norm, vmax


def main():
    run(parse_arguments(), "HapHiC_plot.log")


if __name__ == "__main__":
    main()
