"""Assembly correction (``--correct_nrounds``) of `haphic cluster`: correct_assembly and its helpers
(scripts/HapHiC_cluster.py:943-1536, v1.0.7).

The per-record and per-bin work runs on the GPU (hh_correct_* in libhaphic_b200.so): the coverage pass over the
alignments, breakpoint detection, the coverage / link updates after breaking, and the remapping of the record stream
to the corrected contigs.  The host keeps the bookkeeping of the broken contigs -- piece names, the fa_dict
mutations, sequence slicing, frag_source_dict / final_break_pos_dict / final_break_frag_dict -- with the reference's
dict operations in the reference's insertion orders, and writes corrected_asm.fa / corrected_ctgs.txt.

The alignments are read once: the record batches of the coverage pass are kept and remapped for link counting.
"""

from __future__ import annotations

import ctypes as C
import logging
import os
import time

import numpy as np

from . import _lib
from ._lib import Context, CorrectRoundInfo, check, load, ptr

logger = logging.getLogger("haphic_b200.cluster")


def _records(rec):
    """(records, mem): a numpy int32 [m, 4] array, or a contiguous int32 [m, 4] torch CUDA tensor left on the device."""
    if isinstance(rec, np.ndarray) or not getattr(rec, "is_cuda", False):
        return np.ascontiguousarray(np.asarray(rec), dtype=np.int32).reshape(-1, 4), _lib.HH_MEM_HOST
    import torch
    if rec.dtype != torch.int32 or rec.dim() != 2 or rec.shape[1] != 4 or not rec.is_contiguous():
        raise ValueError("records must be a contiguous int32 [m, 4] tensor")
    torch.cuda.current_stream(rec.device).synchronize()      # the library runs on its own stream
    return rec, _lib.HH_MEM_DEVICE


class Correction:
    """Device state of one correction run (hh_correct): coverage arrays of len//res + 1 bins per contig, the stored
    same-contig links and the fragments under examination."""

    def __init__(self, ctx: Context, ctg_len, resolution: int):
        self.ctx = ctx
        self.resolution = int(resolution)
        self._len = np.ascontiguousarray(ctg_len, dtype=np.int64)
        self.n_ctg = len(self._len)
        self._h = C.c_void_p()
        check(load().hh_correct_create(ctx.handle, self.n_ctg, ptr(self._len), self.resolution, C.byref(self._h)))
        ctx.adopt(self)

    def add(self, rec):
        """Coverage pass over one batch of int32 [m, 4] records (every record may be passed: records of two contigs or of
        contigs outside the FASTA are ignored)."""
        rec, mem = _records(rec)
        if len(rec):
            check(load().hh_correct_add(self._h, ptr(rec), len(rec), mem))

    def round(self, median_cov_ratio, region_len_ratio, min_region_cutoff, last_round):
        """One correction round; returns the CorrectRoundInfo."""
        info = CorrectRoundInfo()
        check(load().hh_correct_round(self._h, float(median_cov_ratio), float(region_len_ratio), int(min_region_cutoff),
                                      int(bool(last_round)), C.byref(info)))
        self.last = info
        return info

    def breaks(self):
        """(fragment id, bin, coverage) of the last round's breakpoints, int32 arrays."""
        n = int(self.last.n_breaks)
        out = [np.empty(n, np.int32) for _ in range(3)]
        if n:
            check(load().hh_correct_fetch_breaks(self._h, *(ptr(a) for a in out)))
        return tuple(out)

    def coverage(self):
        """{fragment id: int32 coverage array} of the fragments under examination, in examination order."""
        n_act, bins = C.c_int32(), C.c_int64()
        check(load().hh_correct_info(self._h, C.byref(n_act), C.byref(bins), None))
        frag = np.empty(n_act.value, np.int32)
        nb = np.empty(n_act.value, np.int32)
        cov = np.empty(max(1, bins.value), np.int32)
        check(load().hh_correct_fetch_cov(self._h, ptr(frag), ptr(nb), ptr(cov)))
        cuts = np.concatenate([[0], np.cumsum(nb.astype(np.int64))])
        return {int(f): cov[cuts[k]:cuts[k + 1]].copy() for k, f in enumerate(frag.tolist())}

    def set_layout(self, src_base, piece_start, piece_id):
        self._layout = (np.ascontiguousarray(src_base, dtype=np.int32), np.ascontiguousarray(piece_start, dtype=np.int64),
                        np.ascontiguousarray(piece_id, dtype=np.int32))
        check(load().hh_correct_set_layout(self._h, *(ptr(a) for a in self._layout), len(self._layout[1])))

    def remap(self, rec, in_place=False):
        """The int32 [m, 4] batch with every end moved to the corrected contigs: a new batch, or ``rec`` itself rewritten
        (``in_place``; saves a fresh host allocation per batch)."""
        rec, mem = _records(rec)
        if in_place:
            out = rec
        else:
            out = np.empty_like(rec) if mem == _lib.HH_MEM_HOST else rec.new_empty(rec.shape)
        if len(rec):
            check(load().hh_correct_remap(self._h, ptr(rec), ptr(out), len(rec), mem))
        return out

    def close(self):
        if self._h:
            load().hh_correct_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------------
# the coverage pass: one read of the alignments, batches kept for the remapped link counting
# ------------------------------------------------------------------------------------------------

def _coverage_pass(corr, batches):
    kept = []
    for rec in batches:
        corr.add(rec)
        kept.append(rec)
    return kept


def parse_pairs_for_correction(corr, batches):
    """1300-1344 (the log line is the reference's)."""
    logger.info("Parsing input pairs file for contig correction...")
    return _coverage_pass(corr, batches)


def parse_bam_for_correction(corr, batches):
    """1362-1398 (the log line is the reference's)."""
    logger.info("Parsing input BAM file for contig correction...")
    return _coverage_pass(corr, batches)


# ------------------------------------------------------------------------------------------------
# host bookkeeping (break_and_update_ctgs 1017-1197, correct_assembly 1200-1297)
# ------------------------------------------------------------------------------------------------

def piece_names(ctg, points, length, unbroken):
    """Names of the pieces of fragment ``ctg`` (``length`` bp) broken at the relative positions ``points`` (ascending):
    '{contig}:{start}-{end}', 1-based inclusive on the source contig (1122-1165)."""
    if ctg in unbroken:
        raw, shift = ctg, 0
    else:
        raw, rng = ctg.rsplit(":", 1)
        shift = int(rng.split("-")[0]) - 1
    bounds = [0] + list(points) + [length]
    return ["{}:{}-{}".format(raw, bounds[k] + 1 + shift, bounds[k + 1] + shift) for k in range(len(bounds) - 1)]


def break_and_update_ctgs(breaks, frag_source, final_pos, final_frag, fa_dict, unbroken, count_RE, new_ids=None,
                          read_depth_dict=None):
    """The fa_dict / break-table part of break_and_update_ctgs (1115-1190).  ``breaks`` = [(ctg, [points])] in
    ctg_break_point_dict order.  ``new_ids`` (list) receives the piece names in the order the device numbers them.  A
    non-empty ``read_depth_dict`` (--gfa) gives every piece its parent's entry and loses the parent's (1147-1149, 1186-1187)."""
    logger.info("Breaking contigs and updating data...")
    for ctg, points in breaks:
        seq, length = fa_dict[ctg][0], fa_dict[ctg][1]
        names = piece_names(ctg, points, length, unbroken)
        source = frag_source[ctg]
        at = final_frag[source].index(ctg)
        father_pos = final_pos[source][at]
        final_frag[source].pop(at)
        final_pos[source].pop(at)
        bounds = [0] + list(points) + [length]
        for k, name in enumerate(names):
            s, e = bounds[k], bounds[k + 1]
            frag_source[name] = source
            final_frag[source].insert(at, name)       # every piece at the father's index: descending starts
            final_pos[source].insert(at, father_pos + s)
            piece = seq[s:e]
            fa_dict[name] = [piece, e - s, count_RE(piece)]   # no +1 pseudo-count here (1031)
            if read_depth_dict:
                read_depth_dict[name] = read_depth_dict[ctg]
            if new_ids is not None:
                new_ids.append(name)
        del fa_dict[ctg]
        if read_depth_dict:
            del read_depth_dict[ctg]


def correct_assembly(corr, fa_dict, args, count_RE, read_depth_dict=None):
    """correct_assembly (1200-1297) on a Correction whose coverage pass is done.  Mutates fa_dict; writes
    corrected_asm.fa and corrected_ctgs.txt; returns (nbroken_ctgs, final_break_pos_dict, final_break_frag_dict)."""
    logger.info("Performing assembly correction...")
    res = int(args.correct_resolution)
    unbroken = set(fa_dict.keys())
    frag_name = list(fa_dict.keys())              # device fragment id -> name
    frag_source, final_pos, final_frag = dict(), dict(), dict()
    nbroken = 0
    for nround in range(args.correct_nrounds):
        last = nround + 1 == args.correct_nrounds
        info = corr.round(args.median_cov_ratio, args.region_len_ratio, args.min_region_cutoff, last)
        logger.info("Correction round {}, breakpoints are detected in {} contig(s)".format(nround + 1, int(info.n_broken)))
        if nround == 0:
            nbroken = int(info.n_broken)
        if not info.n_broken:
            break
        frag, bins, _cov = corr.breaks()
        breaks = []
        for f, b in zip(frag.tolist(), bins.tolist()):
            if not breaks or breaks[-1][0] != frag_name[f]:
                breaks.append((frag_name[f], []))
            breaks[-1][1].append(b * res)
        if nround == 0:
            for ctg, _ in breaks:
                frag_source[ctg] = ctg
                final_pos[ctg] = [0]
                final_frag[ctg] = [ctg]
        new_ids = []
        break_and_update_ctgs(breaks, frag_source, final_pos, final_frag, fa_dict, unbroken, count_RE, new_ids, read_depth_dict)
        if not last:
            assert len(frag_name) == int(info.n_frag)
            frag_name += new_ids
        unbroken -= {ctg for ctg, _ in breaks}
    gfa_list = args.gfa.split(",") if args.gfa else []
    write_corrected_files(fa_dict, unbroken, nbroken, args.fasta,
                          read_depth_dict, gfa_list if args.quick_view and read_depth_dict and len(gfa_list) >= 2 else None)
    return nbroken, final_pos, final_frag


def write_corrected_files(fa_dict, unbroken, nbroken, fasta, read_depth_dict=None, gfa_list=None):
    """corrected_asm.fa / corrected_ctgs.txt (1252-1290); an existing corrected_asm.fa is renamed first.  With ``gfa_list``
    (quick view with >= 2 GFA files) also corrected_<GFA basename> per haplotype for `haphic reassign`: the S lines of the
    corrected contigs of that haplotype in read_depth_dict order, or a symlink to the GFA when nothing was broken."""
    asm_file, list_file = "corrected_asm.fa", "corrected_ctgs.txt"
    logger.info("Generating corrected assembly file...")
    if os.path.exists(asm_file):
        bak = "{}.bak.{}".format(asm_file, time.time())
        logger.info("File {} already exists! Rename it as {}".format(asm_file, bak))
        os.rename(asm_file, bak)
    if nbroken:
        logger.info("{} contigs were broken into {} contigs. Writing corrected assembly to {}...".format(
            nbroken, len(fa_dict) - len(unbroken), asm_file))
        with open(asm_file, "w") as f:
            for ctg, info in fa_dict.items():
                f.write(">{}\n{}\n".format(ctg, info[0]))
        with open(list_file, "w") as f:
            for ctg in fa_dict:
                if ctg not in unbroken:
                    f.write(ctg + "\n")
        for hap, gfa in enumerate(gfa_list or ()):
            with open("corrected_" + os.path.basename(gfa), "w") as f:
                for ctg, (h, depth) in read_depth_dict.items():
                    if h == hap:
                        f.write("S\t{}\t*\tLN:i:{}\trd:i:{}\n".format(ctg, fa_dict[ctg][1], depth))
    else:
        logger.info("No corrected contigs were found. Simply create a symbolic link of the input assembly")
        os.symlink(fasta, asm_file)
        with open(list_file, "w"):
            pass
        for gfa in gfa_list or ():
            os.symlink(gfa, "corrected_" + os.path.basename(gfa))


def remap_layout(src_names, fa_dict, final_pos, final_frag):
    """(src_base, piece_start, piece_id) of hh_correct_set_layout: for every source contig (input FASTA order) its pieces
    by ascending start (final_break_pos_dict lists them descending), ids in the corrected fa_dict."""
    new_id = {n: i for i, n in enumerate(fa_dict)}
    base, starts, ids = [0], [], []
    for ctg in src_names:
        if ctg in final_frag:
            for pos, name in zip(final_pos[ctg][::-1], final_frag[ctg][::-1]):
                starts.append(pos)
                ids.append(new_id[name])
        else:
            starts.append(0)
            ids.append(new_id[ctg])
        base.append(len(starts))
    return np.asarray(base, np.int32), np.asarray(starts, np.int64), np.asarray(ids, np.int32)


def run_correction(ctx, fa_dict, args, batches, count_RE, read_depth_dict=None):
    """The whole correction step of run() (2798-2808, 2835-2851): one read of the alignments feeds the coverage pass;
    returns (record batches for link counting, nbroken_ctgs).  The batches are remapped to the corrected contigs when
    anything was broken, else returned as read."""
    src_names = list(fa_dict.keys())
    corr = Correction(ctx, [fa_dict[n][1] for n in src_names], args.correct_resolution)
    try:
        if args.aln_format == "bam":
            kept = parse_bam_for_correction(corr, batches)
        else:
            kept = parse_pairs_for_correction(corr, batches)
        nbroken, final_pos, final_frag = correct_assembly(corr, fa_dict, args, count_RE, read_depth_dict)
        if nbroken:
            corr.set_layout(*remap_layout(src_names, fa_dict, final_pos, final_frag))
            kept = [corr.remap(rec, in_place=True) for rec in kept]
    finally:
        corr.close()
    return kept, nbroken
