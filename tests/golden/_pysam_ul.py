"""Functional stand-in for the part of `pysam` that the reference's parse_ul_alignments uses, for the golden generator
(make_ul_golden.py) and the host tests.  Pure Python: the BAM is read with gzip (BGZF is multi-member gzip) and decoded
with struct; it shares no code with the native reader.  Attributes follow pysam's documented semantics (AlignedSegment,
pysam 0.22): query_alignment_start / _end as getQueryStart / getQueryEnd, infer_read_length including hard clips.
Only ``format_options=[b'filter=!flag.unmap']`` is understood."""

import gzip
import struct

BAM_CMATCH, BAM_CINS, BAM_CDEL, BAM_CREF_SKIP, BAM_CSOFT_CLIP, BAM_CHARD_CLIP, BAM_CPAD, BAM_CEQUAL, BAM_CDIFF = range(9)
_AUX_SIZE = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4, "d": 8}
_AUX_INT = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I"}


def set_verbosity(_level):
    return 0


class AlignedSegment:
    def __init__(self, header_names, data):
        (self.reference_id, self.reference_start, l_read_name, self.mapping_quality, _bin, n_cigar, self.flag, l_seq,
         _mref, _mpos, _tlen) = struct.unpack_from("<iiBBHHHiiii", data, 0)
        off = 32
        self.query_name = data[off:off + l_read_name - 1].decode()
        off += l_read_name
        raw = struct.unpack_from("<{}I".format(n_cigar), data, off)
        self.cigartuples = [(c & 15, c >> 4) for c in raw]
        off += 4 * n_cigar + (l_seq + 1) // 2 + l_seq
        self._l_qseq = l_seq
        self._aux = data[off:]
        self.reference_name = header_names[self.reference_id] if self.reference_id >= 0 else None

    # flags
    @property
    def mapq(self):
        return self.mapping_quality

    @property
    def is_reverse(self):
        return bool(self.flag & 0x10)

    @property
    def is_forward(self):
        return not self.is_reverse

    @property
    def is_supplementary(self):
        return bool(self.flag & 0x800)

    # coordinates
    @property
    def reference_length(self):
        if not self.cigartuples:
            return None
        return sum(n for op, n in self.cigartuples if op in (BAM_CMATCH, BAM_CDEL, BAM_CREF_SKIP, BAM_CEQUAL, BAM_CDIFF))

    @property
    def reference_end(self):
        return self.reference_start + self.reference_length

    @property
    def query_alignment_start(self):
        start = 0
        for op, n in self.cigartuples:
            if op == BAM_CHARD_CLIP:
                continue
            if op == BAM_CSOFT_CLIP:
                start += n
            else:
                break
        return start

    @property
    def query_alignment_end(self):
        end = self._l_qseq
        if end == 0:
            # no SEQ: the length is taken from the CIGAR (a soft clip only counts while nothing else has)
            for op, n in self.cigartuples:
                if op in (BAM_CMATCH, BAM_CINS, BAM_CEQUAL, BAM_CDIFF) or (op == BAM_CSOFT_CLIP and end == 0):
                    end += n
            return end
        for op, n in reversed(self.cigartuples[1:]):
            if op == BAM_CSOFT_CLIP:
                end -= n
            elif op != BAM_CHARD_CLIP:
                break
        return end

    def infer_read_length(self):
        return sum(n for op, n in self.cigartuples
                   if op in (BAM_CMATCH, BAM_CINS, BAM_CSOFT_CLIP, BAM_CHARD_CLIP, BAM_CEQUAL, BAM_CDIFF))

    def get_tag(self, tag):
        a, off = self._aux, 0
        while off + 3 <= len(a):
            name, typ = a[off:off + 2].decode(), chr(a[off + 2])
            off += 3
            if typ in ("Z", "H"):
                size = a.index(b"\x00", off) - off + 1
            elif typ == "B":
                sub, count = chr(a[off]), struct.unpack_from("<I", a, off + 1)[0]
                size = 5 + count * _AUX_SIZE[sub]
            else:
                size = _AUX_SIZE[typ]
            if name == tag:
                if typ not in _AUX_INT:
                    raise NotImplementedError("only integer tags are decoded")
                return struct.unpack_from(_AUX_INT[typ], a, off)[0]
            off += size
        raise KeyError("tag '{}' not present".format(tag))


class AlignmentFile:
    def __init__(self, path, mode="rb", format_options=None, threads=1):
        assert mode == "rb"
        assert format_options in (None, [b"filter=!flag.unmap"]), format_options
        self._skip_unmapped = format_options is not None
        with gzip.open(path, "rb") as f:
            self._data = f.read()
        d = self._data
        assert d[:4] == b"BAM\x01"
        l_text = struct.unpack_from("<i", d, 4)[0]
        off = 8 + l_text
        n_ref = struct.unpack_from("<i", d, off)[0]
        off += 4
        self.references, self.lengths = [], []
        for _ in range(n_ref):
            l_name = struct.unpack_from("<i", d, off)[0]
            self.references.append(d[off + 4:off + 4 + l_name - 1].decode())
            self.lengths.append(struct.unpack_from("<i", d, off + 4 + l_name)[0])
            off += 8 + l_name
        self._start = off

    def get_reference_length(self, name):
        return self.lengths[self.references.index(name)]

    def __iter__(self):
        d, off = self._data, self._start
        while off < len(d):
            size = struct.unpack_from("<i", d, off)[0]
            aln = AlignedSegment(self.references, d[off + 4:off + 4 + size])
            off += 4 + size
            if self._skip_unmapped and aln.flag & 0x4:
                continue
            yield aln

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False
