"""Alignment readers for the cluster step: .pairs / .pairs.gz text and BAM, yielding int32 record
batches [m, 4] = (ctg_a, pos_a, ctg_b, pos_b) with 0-based positions -- the tuples the reference's
generators yield (scripts/HapHiC_cluster.py:1539-1593) after name -> id translation
(-1 = name not in the FASTA, skipped downstream like HapHiC_cluster.py:1625).

pysam/htslib are not required: both formats are decoded natively (hh_pairs_* / hh_bam_* in
libhaphic_b200.so; BGZF blocks are inflated on several host threads).  A minimal BAM writer is
included for fixtures and tests.
"""

from __future__ import annotations

import gzip
import io
import os
import struct
import zlib

import numpy as np


# ------------------------------------------------------------------------------------------------
# .pairs
# ------------------------------------------------------------------------------------------------

def _open_text(path, aln_format):
    if aln_format == "pairs":
        return open(path, "rt")
    if aln_format == "bgzipped_pairs":
        return gzip.open(path, "rt")
    raise AssertionError("unknown pairs format {!r}".format(aln_format))


def names_blob(names):
    """NUL-terminated concatenation of names for the C ABI."""
    return b"".join(n.encode() + b"\x00" for n in names)


def pairs_batches(path, aln_format, name_to_id, bed_path="alignments.bed", batch_lines=4_000_000, inter_only=True, threads=0):
    """Yield int32 [m, 4] record batches from a 4DN .pairs / .pairs.gz file.

    Mirrors pairs_generator / pairs_generator_inter_ctgs (1539-1583): blank lines and lines starting
    with '#' are skipped; columns are whitespace separated; ``ref, pos, mref, mpos = cols[1],
    int(cols[2])-1, cols[3], int(cols[4])-1``; two BED lines per pair go to ``alignments.bed``
    (needed later by `haphic build` for .pairs input); with ``inter_only`` pairs on one contig are
    dropped (1582).  Tokenising, name lookup and the BED writer are native and multi-threaded (hh_pairs_* in
    libhaphic_b200.so; ``threads`` = 0 uses the host's cores, at most 16); plain gzip streams are inflated by zlib,
    bgzipped files block-parallel."""
    import ctypes as C
    from ._lib import check, load
    assert aln_format in ("pairs", "bgzipped_pairs"), aln_format
    names = name_to_id.names
    blob = names_blob(names)
    h = C.c_void_p()
    lib = load()
    check(lib.hh_pairs_open(os.fsencode(path), blob, len(names), os.fsencode(bed_path) if bed_path else None,
                            int(bool(inter_only)), int(threads), C.byref(h)))
    try:
        n_out = C.c_int64()
        while True:
            rec = np.empty((batch_lines, 4), np.int32)
            check(lib.hh_pairs_next(h, rec.ctypes.data_as(C.c_void_p), batch_lines, C.byref(n_out)))
            m = int(n_out.value)
            if m == 0:
                break
            yield rec[:m]
        check(lib.hh_pairs_close(h))          # reports a failed alignments.bed write
        h = None
    finally:
        if h is not None:
            lib.hh_pairs_close(h)


class NameIndex:
    """The contig names in id order (= FASTA order) with a name -> id lookup (-1 = unknown)."""

    def __init__(self, names):
        self.names = list(names)
        self._d = {n: i for i, n in enumerate(self.names)}

    def __getitem__(self, name):
        return self._d.get(name, -1)


# ------------------------------------------------------------------------------------------------
# BAM
# ------------------------------------------------------------------------------------------------

class BamHeader:
    def __init__(self, text, ref_names, ref_lengths):
        self.text = text
        self.ref_names = ref_names
        self.ref_lengths = ref_lengths

    @property
    def sort_order(self):
        for line in self.text.splitlines():
            if line.startswith("@HD"):
                for tok in line.split("\t")[1:]:
                    if tok.startswith("SO:"):
                        return tok[3:]
        return None


def _read_exact(f, n):
    b = f.read(n)
    if len(b) != n:
        raise EOFError("truncated BAM")
    return b


def read_bam_header(f):
    if _read_exact(f, 4) != b"BAM\x01":
        raise RuntimeError("not a BAM file")
    (l_text,) = struct.unpack("<i", _read_exact(f, 4))
    text = _read_exact(f, l_text).rstrip(b"\x00").decode()
    (n_ref,) = struct.unpack("<i", _read_exact(f, 4))
    names, lens = [], []
    for _ in range(n_ref):
        (l_name,) = struct.unpack("<i", _read_exact(f, 4))
        names.append(_read_exact(f, l_name)[:-1].decode())
        lens.append(struct.unpack("<i", _read_exact(f, 4))[0])
    return BamHeader(text, names, lens)


def bam_batches(path, name_to_id, inter_only=True, batch_records=4_000_000, logger=None, threads=0):
    """Yield int32 [m, 4] record batches from a BAM file: one record per read1 alignment
    (``flag.read1``; plus ``refid != mrefid`` with ``inter_only`` -- the htslib filter strings at
    HapHiC_cluster.py:2855/2862), fields (reference_name, reference_start, next_reference_name,
    next_reference_start) as in bam_generator (1586-1593).  Sorting order is checked like
    check_sorting_order (1347-1359).  BGZF inflation and the record walk are native (hh_bam_* in
    libhaphic_b200.so, `threads` inflate threads; 0 = the host's cores, at most 16)."""
    import ctypes as C
    from ._lib import check, load
    lib = load()
    names = name_to_id.names
    if threads <= 0:
        threads = max(1, min(16, os.cpu_count() or 1))
    h = C.c_void_p()
    check(lib.hh_bam_open(os.fsencode(path), names_blob(names), len(names), int(bool(inter_only)), int(threads), C.byref(h)))
    try:
        text, ln = C.c_char_p(), C.c_int64()
        check(lib.hh_bam_header_text(h, C.byref(text), C.byref(ln)))
        so = BamHeader(C.string_at(text, ln.value).decode(), None, None).sort_order
        if so in ("unsorted", "queryname"):
            if logger:
                logger.info("The sorting order of the BAM file is {}".format(so))
        elif so == "coordinate":
            msg = "The sorting order of the BAM file is {}. It should be unsorted or name-sorted".format(so)
            if logger:
                logger.error(msg)
            raise RuntimeError(msg)
        elif logger:
            logger.warning("The sorting order of the BAM file is unknown, but the program will continue")
        n_out = C.c_int64()
        while True:
            rec = np.empty((batch_records, 4), np.int32)
            check(lib.hh_bam_next(h, rec.ctypes.data_as(C.c_void_p), batch_records, C.byref(n_out)))
            m = int(n_out.value)
            if m == 0:
                break
            yield rec[:m]
    finally:
        lib.hh_bam_close(h)


def _bgzf_block(data: bytes) -> bytes:
    comp = zlib.compressobj(6, zlib.DEFLATED, -15)
    body = comp.compress(data) + comp.flush()
    bsize = len(body) + 25
    hdr = struct.pack("<BBBBIBBHBBHH", 0x1F, 0x8B, 8, 4, 0, 0, 0xFF, 6, ord("B"), ord("C"), 2, bsize)
    return hdr + body + struct.pack("<II", zlib.crc32(data) & 0xFFFFFFFF, len(data) & 0xFFFFFFFF)


def write_bam(path, ref_names, ref_lengths, records, sort_order="unsorted", read_len=50):
    """Minimal paired-end BAM writer for fixtures: ``records`` is an int array [P, 4] of
    (ctg_a, pos_a, ctg_b, pos_b); each pair becomes a read1 and a read2 record with mate fields."""
    out = io.BytesIO()
    text = "@HD\tVN:1.6\tSO:{}\n".format(sort_order) + "".join(
        "@SQ\tSN:{}\tLN:{}\n".format(n, l) for n, l in zip(ref_names, ref_lengths))
    tb = text.encode()
    out.write(b"BAM\x01" + struct.pack("<i", len(tb)) + tb + struct.pack("<i", len(ref_names)))
    for n, l in zip(ref_names, ref_lengths):
        nb = n.encode() + b"\x00"
        out.write(struct.pack("<i", len(nb)) + nb + struct.pack("<i", int(l)))
    seq = bytes([0x11] * ((read_len + 1) // 2))      # 'A' * read_len, 4-bit packed
    qual = bytes([0xFF] * read_len)
    cigar = struct.pack("<I", (read_len << 4) | 0)   # read_len M
    for r, (a, pa, b, pb) in enumerate(np.asarray(records).tolist()):
        name = "r{}".format(r).encode() + b"\x00"
        for (rid, pos, mrid, mpos, flag) in ((a, pa, b, pb, 0x1 | 0x40), (b, pb, a, pa, 0x1 | 0x80)):
            core = struct.pack("<iiBBHHHiiii", rid, pos, len(name), 60, 4680, 1, flag, read_len, mrid, mpos, 0)
            body = core + name + cigar + seq + qual
            out.write(struct.pack("<i", len(body)) + body)
    raw = out.getvalue()
    with open(path, "wb") as f:
        for i in range(0, len(raw), 0xFF00):
            f.write(_bgzf_block(raw[i:i + 0xFF00]))
        f.write(_bgzf_block(b""))


_AS_FMT = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I"}
_CIGAR_OPS = "MIDNSHP=X"


def write_ul_bam(path, ref_names, ref_lengths, records, repeat=1, random_seq=None):
    """Single-end BAM writer for ultra-long read fixtures.  Every record is a dict: ``name``, ``flag``, ``ref`` (index, -1 =
    none), ``pos`` (0-based), ``mapq``, ``cigar`` (a string such as "500S12000M300H"), ``seq`` (False writes SEQ as `*`,
    i.e. l_seq = 0) and optionally ``AS`` = (value, aux type among c C s S i I).  ``repeat`` writes the compressed records
    that many times (large files for throughput measurements); ``random_seq`` (a numpy Generator) fills SEQ and QUAL with
    random bases and qualities, which compress about as well as real reads do (a constant SEQ would not)."""
    import re
    out = io.BytesIO()
    text = "@HD\tVN:1.6\tSO:unsorted\n" + "".join("@SQ\tSN:{}\tLN:{}\n".format(n, l) for n, l in zip(ref_names, ref_lengths))
    tb = text.encode()
    out.write(b"BAM\x01" + struct.pack("<i", len(tb)) + tb + struct.pack("<i", len(ref_names)))
    for n, l in zip(ref_names, ref_lengths):
        nb = n.encode() + b"\x00"
        out.write(struct.pack("<i", len(nb)) + nb + struct.pack("<i", int(l)))
    header = out.getvalue()
    out = io.BytesIO()
    for r in records:
        ops = [(int(ln), _CIGAR_OPS.index(op)) for ln, op in re.findall(r"(\d+)([MIDNSHP=X])", r["cigar"])]
        l_seq = sum(ln for ln, op in ops if op in (0, 1, 4, 7, 8)) if r.get("seq", True) else 0
        name = r["name"].encode() + b"\x00"
        core = struct.pack("<iiBBHHHiiii", int(r["ref"]), int(r["pos"]), len(name), int(r["mapq"]), 4680, len(ops), int(r["flag"]),
                           l_seq, -1, -1, 0)
        cigar = b"".join(struct.pack("<I", (ln << 4) | op) for ln, op in ops)
        if random_seq is None:
            seq = bytes([0x11] * ((l_seq + 1) // 2)) + bytes([0xFF] * l_seq)
        else:
            codes = np.array([1, 2, 4, 8], np.uint8)[random_seq.integers(0, 4, 2 * ((l_seq + 1) // 2))]
            seq = ((codes[0::2] << 4) | codes[1::2]).tobytes() + random_seq.integers(0, 41, l_seq).astype(np.uint8).tobytes()
        aux = b""
        if r.get("AS") is not None:
            value, typ = r["AS"]
            aux = b"AS" + typ.encode() + struct.pack(_AS_FMT[typ], int(value))
        body = core + name + cigar + seq + aux
        out.write(struct.pack("<i", len(body)) + body)
    raw = out.getvalue()
    body = b"".join(_bgzf_block(raw[i:i + 0xFF00]) for i in range(0, len(raw), 0xFF00))
    with open(path, "wb") as f:
        for i in range(0, len(header), 0xFF00):
            f.write(_bgzf_block(header[i:i + 0xFF00]))
        for _ in range(repeat):
            f.write(body)
        f.write(_bgzf_block(b""))
