"""Synthetic Hi-C inputs for tests and bench (SURVEY.md section 8(d)).

Nothing here is on the product path: it only fabricates inputs with the
shape the reference's own simulation tooling produces
(simulation/sim_contigs.py:43-104 names contigs
``{Chrom}_{n}_{start}_{end}_{ori}_{len}``), so that truth can be recovered
from contig names the way simulation/result_statistics.py does.

Model
-----
* ``nchr`` chromosomes of equal length; contigs are cut left to right with
  lengths ~ Normal(mean, 0.3*mean) truncated at >= ``min_len``; orientation is
  Bernoulli(0.5).
* read pairs: with probability ``cis_frac`` both ends fall on one chromosome,
  the first uniformly, the second at a genomic separation drawn from
  P(s) ~ 1/s on [1 kb, chrom_len] (reflected into the chromosome); otherwise
  both ends are uniform over the whole genome.
* a pair record is ``(ctg_a, pos_a, ctg_b, pos_b)`` int32, positions 0-based
  on the contig *as assembled* (i.e. reversed for '-' contigs) -- exactly the
  tuple the reference's generators yield (HapHiC_cluster.py:1562-1593) after
  name -> id translation.  Intra-contig pairs are left in the stream: dropping
  them (``ref != mref``, HapHiC_cluster.py:1582) is part of the path under test.
"""

from __future__ import annotations

import dataclasses
import math

import numpy as np
import torch


@dataclasses.dataclass
class Assembly:
    names: list            # contig names, FASTA order
    lengths: np.ndarray    # int64 [n]
    chrom: np.ndarray      # int32 [n] chromosome of each contig
    start: np.ndarray      # int64 [n] 0-based start of the contig on its chromosome
    ori: np.ndarray        # int8  [n] 1 = reverse-complemented
    chrom_len: int
    nchr: int

    @property
    def n(self) -> int:
        return len(self.names)


def make_assembly(nchr: int, n_contigs: int, mean_len: int, seed: int = 12345,
                  min_len: int = 5000, cv: float = 0.3, prefix: str = "Chr") -> Assembly:
    """Cut ``nchr`` equal chromosomes into ~``n_contigs`` contigs in total."""
    rng = np.random.default_rng(seed)
    per_chr = max(1, n_contigs // nchr)
    chrom_len = per_chr * mean_len
    names, lengths, chrom, start, ori = [], [], [], [], []
    for c in range(nchr):
        # draw lengths until the chromosome is covered, then fix the tail so the
        # chromosome holds exactly ``per_chr`` contigs (keeps n deterministic)
        draw = rng.normal(mean_len, cv * mean_len, size=per_chr * 3).astype(np.int64)
        draw = draw[draw >= min_len][:per_chr]
        assert len(draw) == per_chr, "not enough contig lengths drawn"
        scale = chrom_len / draw.sum()
        lens = np.maximum((draw * scale).astype(np.int64), min_len)
        lens[-1] += chrom_len - lens.sum()
        if lens[-1] < min_len:       # push the deficit into the longest contig
            k = int(np.argmax(lens[:-1]))
            lens[k] -= (min_len - lens[-1])
            lens[-1] = min_len
        assert lens.sum() == chrom_len and (lens > 0).all()
        p = 0
        oris = rng.integers(0, 2, size=per_chr)
        for k, (ln, o) in enumerate(zip(lens.tolist(), oris.tolist()), 1):
            names.append("{}{}_{}_{}_{}_{}_{}".format(prefix, c + 1, k, p + 1, p + ln, "-" if o else "+", ln))
            lengths.append(ln)
            chrom.append(c)
            start.append(p)
            ori.append(o)
            p += ln
    return Assembly(names, np.asarray(lengths, np.int64), np.asarray(chrom, np.int32),
                    np.asarray(start, np.int64), np.asarray(ori, np.int8), int(chrom_len), nchr)


def make_pairs_range(asm: Assembly, lo: int, hi: int, seed: int = 12345, cis_frac: float = 0.85,
                     device: str | torch.device = "cpu", block: int = 1 << 22) -> torch.Tensor:
    """Records [lo, hi) of the (conceptually infinite) pair stream of ``seed``.  The stream is generated in
    independently seeded blocks, so any slicing -- one GPU taking everything, or N ranks taking contiguous
    shards -- sees exactly the same records."""
    parts = []
    b0, b1 = lo // block, (hi + block - 1) // block
    for b in range(b0, b1):
        blk = make_pairs(asm, block, seed=seed * 1000003 + b, cis_frac=cis_frac, device=device, chunk=block)
        s, e = max(lo, b * block) - b * block, min(hi, (b + 1) * block) - b * block
        parts.append(blk[s:e])
    if not parts:
        return torch.empty((0, 4), dtype=torch.int32, device=torch.device(device))
    return torch.cat(parts) if len(parts) > 1 else parts[0].contiguous()


def make_pairs(asm: Assembly, n_pairs: int, seed: int = 12345, cis_frac: float = 0.85,
               device: str | torch.device = "cpu", chunk: int = 1 << 24, homolog=None) -> torch.Tensor:
    """Return an int32 tensor [n_pairs, 4] of (ctg_a, pos_a, ctg_b, pos_b).

    ``homolog=(ploidy, frac)`` treats every ``ploidy`` consecutive chromosomes as the haplotypes of one
    chromosome (as simulation/sim_haplotypes.py lays them out) and re-maps the second end of a fraction ``frac`` of
    the cis pairs to the SAME locus (+- 500 bp) of another haplotype -- the collinear "allelic" Hi-C links that
    remove_allelic_HiC_links (HapHiC_cluster.py:474-692) detects by their concordance ratio."""
    dev = torch.device(device)
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    L = asm.chrom_len
    nchr = asm.nchr
    # contigs are laid out chromosome by chromosome: genome coordinate = chrom*L + pos
    gstart = torch.as_tensor(asm.chrom.astype(np.int64) * L + asm.start, device=dev)
    glen = torch.as_tensor(asm.lengths, device=dev)
    gori = torch.as_tensor(asm.ori.astype(np.int64), device=dev)
    out = torch.empty((n_pairs, 4), dtype=torch.int32, device=dev)
    log_ratio = math.log(L / 1000.0)

    def locate(gpos):
        idx = torch.searchsorted(gstart, gpos, right=True) - 1
        off = gpos - gstart[idx]
        ln = glen[idx]
        off = torch.where(gori[idx] == 1, ln - 1 - off, off)
        return idx.to(torch.int32), off.to(torch.int32)

    done = 0
    while done < n_pairs:
        m = min(chunk, n_pairs - done)
        u = torch.rand((m, 5 if homolog is None else 8), generator=g, device=dev, dtype=torch.float64)
        is_cis = u[:, 0] < cis_frac
        chrom_a = torch.clamp((u[:, 1] * nchr).long(), max=nchr - 1)
        pos_a = torch.clamp((u[:, 2] * L).long(), max=L - 1)
        # cis mate: separation ~ 1/s on [1e3, L], random direction, reflected into [0, L)
        sep = (1000.0 * torch.exp(u[:, 3] * log_ratio)).long()
        sign = torch.where(u[:, 4] < 0.5, -1, 1)
        pos_c = pos_a + sign * sep
        pos_c = torch.where(pos_c < 0, -pos_c, pos_c)
        pos_c = torch.where(pos_c >= L, 2 * (L - 1) - pos_c, pos_c)
        pos_c = torch.clamp(pos_c, 0, L - 1)
        # trans mate: uniform over the genome (re-using u[:,3], u[:,4] as fresh uniforms)
        chrom_t = torch.clamp((u[:, 3] * nchr).long(), max=nchr - 1)
        pos_t = torch.clamp((u[:, 4] * L).long(), max=L - 1)
        g_a = chrom_a * L + pos_a
        g_b = torch.where(is_cis, chrom_a * L + pos_c, chrom_t * L + pos_t)
        if homolog is not None:
            ploidy, frac = int(homolog[0]), float(homolog[1])
            switch = is_cis & (u[:, 5] < frac)
            hap = chrom_a % ploidy
            other = (hap + 1 + torch.clamp((u[:, 6] * (ploidy - 1)).long(), max=ploidy - 2)) % ploidy
            pos_h = torch.clamp(pos_a + ((u[:, 7] - 0.5) * 1000.0).long(), 0, L - 1)
            g_b = torch.where(switch, (chrom_a - hap + other) * L + pos_h, g_b)
        ia, pa = locate(g_a)
        ib, pb = locate(g_b)
        out[done:done + m, 0] = ia
        out[done:done + m, 1] = pa
        out[done:done + m, 2] = ib
        out[done:done + m, 3] = pb
        done += m
    return out


def random_sequence(length: int, rng: np.random.Generator) -> str:
    return "".join(np.array(list("ACGT"))[rng.integers(0, 4, size=length)])


def write_fasta(asm: Assembly, path: str, seed: int = 12345, width: int = 0) -> None:
    """i.i.d. uniform ACGT sequence per contig (GATC every ~256 bp)."""
    rng = np.random.default_rng(seed)
    alphabet = np.frombuffer(b"ACGT", dtype=np.uint8)
    with open(path, "w") as f:
        for name, ln in zip(asm.names, asm.lengths.tolist()):
            seq = alphabet[rng.integers(0, 4, size=ln)].tobytes().decode()
            f.write(">{}\n".format(name))
            if width:
                for i in range(0, ln, width):
                    f.write(seq[i:i + width] + "\n")
            else:
                f.write(seq + "\n")


def write_pairs(asm: Assembly, pairs: np.ndarray, path: str) -> None:
    """4DN .pairs text, 1-based positions, 7 columns (readID chr1 pos1 chr2 pos2 strand1 strand2)."""
    names = asm.names
    with open(path, "w") as f:
        f.write("## pairs format v1.0\n#columns: readID chr1 pos1 chr2 pos2 strand1 strand2\n")
        for r, (a, pa, b, pb) in enumerate(pairs.tolist()):
            f.write("r{}\t{}\t{}\t{}\t{}\t+\t-\n".format(r, names[a], pa + 1, names[b], pb + 1))


def make_chimeras(asm: Assembly, pairs: np.ndarray, joins, span: int = 0, seed: int = 12345, window: int = 2000,
                  gap: int = 0):
    """Misjoined assemblies for assembly correction (``--correct_nrounds``): every tuple of contig ids in ``joins`` is
    joined left to right into one contig named ``chimera{k}``; the joined contigs leave the FASTA and the chimeras follow
    the remaining contigs.  ``pairs`` (int [P, 4]) is mapped onto the new contigs.

    A junction bin always holds the ends of both joined contigs, so their own intra-contig pairs cover it: a plain junction
    is a shallow valley, not an empty one.  ``gap`` > 0 drops every same-chimera record whose span [lo, hi] meets
    [junction - gap, junction + gap) -- the bins inside that window get coverage 0 (a zero-coverage valley; with
    gap >= 2 * resolution at least three bins).  ``span`` > 0 then appends, per junction, that many records with one end in
    the ``window`` bp before the junction and one after it (a valley with non-zero coverage).
    Returns (assembly, pairs, junctions) with junctions = [(chimera id, junction position)]."""
    rng = np.random.default_rng(seed)
    joined = {c for j in joins for c in j}
    keep = [c for c in range(asm.n) if c not in joined]
    new_id = np.full(asm.n, -1, np.int64)
    offset = np.zeros(asm.n, np.int64)
    new_id[keep] = np.arange(len(keep))
    names = [asm.names[c] for c in keep]
    lengths = [int(asm.lengths[c]) for c in keep]
    junctions = []
    for k, group in enumerate(joins):
        cid = len(names)
        at = 0
        for m, c in enumerate(group):
            if m:
                junctions.append((cid, at))
            new_id[c] = cid
            offset[c] = at
            at += int(asm.lengths[c])
        names.append("chimera{}".format(k + 1))
        lengths.append(at)
    p = np.asarray(pairs, np.int64)
    out = np.stack([new_id[p[:, 0]], p[:, 1] + offset[p[:, 0]], new_id[p[:, 2]], p[:, 3] + offset[p[:, 2]]], axis=1)
    if gap > 0 and junctions:
        cand = np.nonzero((out[:, 0] == out[:, 2]) & (out[:, 0] >= len(keep)))[0]
        lo = np.minimum(out[cand, 1], out[cand, 3])
        hi = np.maximum(out[cand, 1], out[cand, 3])
        drop = np.zeros(len(cand), bool)
        for cid, pos in junctions:
            drop |= (out[cand, 0] == cid) & (lo < pos + gap) & (hi >= pos - gap)
        out = np.delete(out, cand[drop], axis=0)
    extra = []
    for cid, pos in junctions:
        for _ in range(span):
            extra.append((cid, pos - 1 - int(rng.integers(0, window)), cid, pos + int(rng.integers(0, window))))
    if extra:
        out = np.concatenate([out, np.asarray(extra, np.int64)])
    n = len(names)
    new = Assembly(names, np.asarray(lengths, np.int64), np.zeros(n, np.int32), np.zeros(n, np.int64), np.zeros(n, np.int8),
                   asm.chrom_len, asm.nchr)
    return new, out.astype(np.int32), junctions


def chimera_case(nchr: int, n_contigs: int, mean_len: int, n_pairs: int, n_joins: int, span: int, seed: int, group: int = 2,
                 device: str = "cpu", gap: int = 1000):
    """A seeded misjoined assembly: ``n_joins`` chimeras of ``group`` contigs, each from another chromosome than the one
    before it.  The first half has ``span`` planted spanning records per junction (non-zero valleys); in the second half
    every junction is a zero-coverage gap of +- ``gap`` bp (make_chimeras).  Returns (assembly, pairs, junctions)."""
    asm = make_assembly(nchr, n_contigs, mean_len, seed=seed)
    pairs = make_pairs(asm, n_pairs, seed=seed + 1, device=device).cpu().numpy()
    rng = np.random.default_rng(seed + 2)
    per_chr = asm.n // nchr
    picks = rng.permutation(per_chr)[:group * n_joins]
    joins = [tuple(int(picks[group * k + m]) + per_chr * ((m * (1 + k % (nchr - 1))) % nchr) for m in range(group))
             for k in range(n_joins)]
    a1, p1, j1 = make_chimeras(asm, pairs, joins[:n_joins // 2], span=span, seed=seed + 3)
    if n_joins // 2 == n_joins:
        return a1, p1, j1
    # the second half: zero-coverage junctions (ids refer to the first result's contigs, whose order is preserved)
    ids = {nm: i for i, nm in enumerate(a1.names)}
    joins2 = [tuple(ids[asm.names[c]] for c in j) for j in joins[n_joins // 2:]]
    a2, p2, j2 = make_chimeras(a1, p1, joins2, span=0, seed=seed + 4, gap=gap)
    moved = {i: a2.names.index(a1.names[i]) for i, _ in j1}
    for k in range(len(joins2)):
        a2.names[-(len(joins2) - k)] = "chimera{}".format(n_joins // 2 + k + 1)
    return a2, p2, [(moved[c], pos) for c, pos in j1] + j2


def write_gfa(asm: Assembly, paths, seed: int = 12345, depth: int = 30, collapsed: int = 4, extra=(), hap=None,
              ploidy=None) -> np.ndarray:
    """hifiasm-style GFA files of a haplotype-resolved assembly, one per haplotype: contig c belongs to haplotype
    ``hap[c]`` (default ``chrom[c] % ploidy``, the layout of make_pairs(homolog=(ploidy, ...)); ploidy defaults to
    ``len(paths)``) and goes to file ``hap[c] % len(paths)`` -- one file holds every contig -- as an ``S name * LN:i: rd:i:``
    line followed by one ``A`` line; every file ends with ``L`` lines between its consecutive contigs.  Read depths are
    ``depth`` +- 20 %, except for ``collapsed`` contigs at 2-3x (collapsed repeats, the outliers of the read-depth filter).
    ``extra`` names contigs written to the first file only (GFA segments missing from the FASTA).  Returns the depths."""
    rng = np.random.default_rng(seed)
    nfile = len(paths)
    ploidy = ploidy or nfile
    if hap is None:
        hap = asm.chrom.astype(np.int64) % ploidy
    rd = rng.integers(int(depth * 0.8), int(depth * 1.2) + 1, size=asm.n)
    if collapsed:
        pick = rng.choice(asm.n, size=min(collapsed, asm.n), replace=False)
        rd[pick] *= rng.integers(2, 4, size=len(pick))
    files = [open(p, "w") for p in paths]
    try:
        for f in files:
            f.write("H\tVN:Z:1.0\n")
        last = [None] * nfile
        links = [[] for _ in range(nfile)]
        for c, (name, ln) in enumerate(zip(asm.names, asm.lengths.tolist())):
            h = int(hap[c]) % nfile
            files[h].write("S\t{}\t*\tLN:i:{}\trd:i:{}\n".format(name, ln, int(rd[c])))
            files[h].write("A\t{}\t0\t+\tread{}\t0\t{}\tid:i:{}\tHG:A:*\n".format(name, c, min(ln, 20000), c))
            if last[h] is not None:
                links[h].append("L\t{}\t+\t{}\t+\t0M\tL1:i:{}\n".format(last[h], name, ln))
            last[h] = name
        for k, name in enumerate(extra):
            files[0].write("S\t{}\t*\tLN:i:{}\trd:i:{}\n".format(name, 10000 + k, depth))
        for f, ls in zip(files, links):
            f.writelines(ls)
    finally:
        for f in files:
            f.close()
    return rd


def gfa_case(nchr, n_contigs, mean_len, n_pairs, seed, ploidy, n_gfa, chimeras, out_dir, bam=False):
    """A seeded haplotype-resolved input set for `haphic cluster --gfa` in ``out_dir``: asm.fa, aln.pairs (or aln.bam) and
    h1.gfa .. h{n_gfa}.gfa.  ``nchr`` chromosomes form nchr / ploidy homologous groups (make_pairs(homolog=(ploidy, 0.2)));
    ``chimeras`` > 0 joins that many pairs of contigs of one haplotype (for --correct_nrounds).  Returns the GFA paths."""
    import os
    asm = make_assembly(nchr, n_contigs, mean_len, seed=seed)
    pairs = make_pairs(asm, n_pairs, seed=seed + 1, homolog=(ploidy, 0.2)).numpy()
    hap = None
    if chimeras:
        rng = np.random.default_rng(seed + 2)
        per = asm.n // nchr
        joins = [(int(c), int(c) + per * ploidy) for c in rng.permutation(per)[:chimeras]]
        joined = {x for j in joins for x in j}
        # make_chimeras keeps the other contigs in order and appends the chimeras
        hap = np.array([int(asm.chrom[c]) % ploidy for c in range(asm.n) if c not in joined]
                       + [int(asm.chrom[j[0]]) % ploidy for j in joins], np.int32)
        asm, pairs, _ = make_chimeras(asm, pairs, joins, seed=seed + 3, gap=1000)
    write_fasta(asm, os.path.join(out_dir, "asm.fa"), seed=seed + 3)
    if bam:
        from . import hicio
        hicio.write_bam(os.path.join(out_dir, "aln.bam"), asm.names, asm.lengths.tolist(), pairs)
    else:
        write_pairs(asm, pairs, os.path.join(out_dir, "aln.pairs"))
    gfa = [os.path.join(out_dir, "h{}.gfa".format(k + 1)) for k in range(n_gfa)]
    write_gfa(asm, gfa, seed=seed + 4, hap=hap, ploidy=ploidy)
    return gfa


def _ul_cigar(q0, q1, read_len, reverse, clip):
    """CIGAR of an alignment of query [q0, q1) of a read of ``read_len`` bases (reverse: in reference orientation)."""
    left, right = (read_len - q1, q0) if reverse else (q0, read_len - q1)
    return "".join("{}{}".format(n, op) for n, op in ((left, clip), (q1 - q0, "M"), (right, clip)) if n)


def ul_read(name, a, b, read_no=0, gap=50, span=12000, as_types="iI", rng=None):
    """Records of one ultra-long read across a junction: ``a`` and ``b`` are (ref index, ref length, reverse) of the two
    parts in read order.  The primary is one part (a, or b when ``read_no`` is odd), the supplementary the other, with
    SEQ `*`; the first part is soft-clipped, a forward supplementary sometimes hard-clipped."""
    rng = rng or np.random.default_rng(read_no)
    m_a, m_b = min(span, a[1]), min(span, b[1])
    qa = (100, 100 + m_a)
    qb = (qa[1] + gap, qa[1] + gap + m_b)
    read_len = qb[1] + 100
    parts = []
    for k, ((ref, ln, rev), q, m, first) in enumerate(((a, qa, m_a, True), (b, qb, m_b, False))):
        # the first part of the read sits at its contig's right end when forward, the second at the left end
        pos = (ln - m if not rev else 0) if first else (0 if not rev else ln - m)
        parts.append(dict(ref=ref, pos=pos, q=q, rev=rev))
    prim, supp = (parts[1], parts[0]) if read_no % 2 else (parts[0], parts[1])
    hard = not supp["rev"] and rng.random() < 0.5
    recs = [dict(name=name, flag=16 if prim["rev"] else 0, ref=prim["ref"], pos=prim["pos"], mapq=60,
                 cigar=_ul_cigar(*prim["q"], read_len, prim["rev"], "S"), seq=True, AS=(int(rng.integers(0, 30000)), "i")),
            dict(name=name, flag=0x800 | (0x10 if supp["rev"] else 0), ref=supp["ref"], pos=supp["pos"], mapq=60,
                 cigar=_ul_cigar(*supp["q"], read_len, supp["rev"], "H" if hard else "S"), seq=hard,
                 AS=(int(rng.integers(0, 120)), str(rng.choice(list(as_types)))))]
    return recs


def ul_reads(asm, seed, support=3, keep=0.7, detour=None):
    """Ultra-long reads across the junctions of consecutive contigs of every chromosome: a junction is covered with
    probability ``keep`` by ``support`` reads (one read, below the default --min_ul_support, otherwise).  Every contig
    keeps one strand (its orientation), so the semi-contig edges of a chromosome form a chain.  ``detour`` = (contig,
    length) routes the first covered junction through an extra BAM reference of that name that is not in the FASTA.
    Returns (reference names, reference lengths, records)."""
    rng = np.random.default_rng(seed)
    names, lengths = list(asm.names), [int(x) for x in asm.lengths.tolist()]
    if detour:
        names.append(detour[0])
        lengths.append(int(detour[1]))
    recs = []
    n_read = 0
    for c in range(asm.n - 1):
        if asm.chrom[c] != asm.chrom[c + 1]:
            continue
        a = (c, lengths[c], bool(asm.ori[c]))
        b = (c + 1, lengths[c + 1], bool(asm.ori[c + 1]))
        hops = [(a, b)]
        if detour and n_read == 0:
            x = (len(names) - 1, lengths[-1], False)
            hops = [(a, x), (x, b)]
        n_reads = support if rng.random() < keep else 1
        for a_, b_ in hops:
            for _ in range(n_reads):
                recs += ul_read("ul{}".format(n_read), a_, b_, read_no=n_read, rng=rng)
                n_read += 1
    return names, lengths, recs


def ul_case(nchr, n_contigs, mean_len, n_pairs, seed, out_dir, ploidy=1, n_gfa=0, bam=False, no_path=False):
    """A seeded input set for `haphic cluster --ul` in ``out_dir``: asm.fa, aln.pairs (or aln.bam), ul.bam and, with
    ``n_gfa``, h1.gfa .. (gfa_case).  ``no_path`` writes UL reads that support no junction.  Returns the GFA paths."""
    import os
    from . import hicio
    gfa = gfa_case(nchr, n_contigs, mean_len, n_pairs, seed, max(1, ploidy), max(1, n_gfa), 0, out_dir, bam=bam)
    if not n_gfa:
        for p in gfa:
            os.remove(p)
        gfa = []
    asm = make_assembly(nchr, n_contigs, mean_len, seed=seed)
    names, lengths, recs = ul_reads(asm, seed + 7, support=1 if no_path else 3, detour=("ul_unplaced_1", 30000))
    hicio.write_ul_bam(os.path.join(out_dir, "ul.bam"), names, lengths, recs)
    return gfa


def _ul_rec(name, part, read_len, flag_extra=0, clip="S", seq=True):
    return dict(name=name, flag=flag_extra | (0x10 if part["rev"] else 0), ref=part["ref"], pos=part["pos"],
                mapq=part.get("mapq", 60), cigar=_ul_cigar(*part["q"], read_len, part["rev"], clip), seq=seq,
                AS=part.get("AS", (1000, "i")))


def ul_adversarial():
    """(reference names, lengths, records) of UL alignments at the edges of parse_ul_alignments: every filter just on
    either side of its threshold (MAPQ 30 / 29, length 10000 / 9999, end distance 100 / 101, overlap ratio 0.5 / above,
    gap 10000 / 10001 -- each as the second of two reads, so it decides whether the pair reaches the default support of 2),
    AS ties over mixed aux widths, supplementaries on the primary's contig, before their primary and after a failed
    primary, secondary / unmapped / reverse-supplementary flags, a contig reached from three sides, a ring whose inter
    edges tie for the lightest, junctions below the support, names with `_` and `_bin`, and a path through a reference
    that the FASTA lacks."""
    names = ["a_1", "b_1", "c_bin1", "d_bin", "rep", "e", "f", "g", "r0", "r1", "r2", "r3", "h", "i", "w1", "noFA", "w2"]
    tests = ["mapq", "len", "dist", "overlap", "gap"]
    for t in tests:
        for side in ("pass", "fail"):
            names += ["{}_{}_p".format(t, side), "{}_{}_q".format(t, side)]
    names += ["tie_p", "tie_q", "tie_z"]
    lengths = [50000] * len(names)
    ix = {n: k for k, n in enumerate(names)}
    rng = np.random.default_rng(77)
    recs = []
    count = [0]

    def junction(x, y, n=3, rev=(False, False)):
        for _ in range(n):
            recs.extend(ul_read("j{}".format(count[0]), (ix[x], 50000, rev[0]), (ix[y], 50000, rev[1]), read_no=count[0],
                                as_types="cCsSiI", rng=rng))
            count[0] += 1

    for x, y in (("a_1", "b_1"), ("b_1", "c_bin1"), ("c_bin1", "d_bin")):
        junction(x, y, rev=(x == "b_1", False))
    for x in ("e", "f", "g"):
        junction(x, "rep")
    for x, y in (("r0", "r1"), ("r1", "r2"), ("r2", "r3"), ("r3", "r0")):
        junction(x, y)
    junction("h", "i", n=1)
    junction("w1", "noFA")
    junction("noFA", "w2")

    def pair_read(name, p, s, extra=()):
        read_len = max(p["q"][1], s["q"][1]) + 100
        recs.append(_ul_rec(name, p, read_len))
        recs.append(_ul_rec(name, s, read_len, 0x800, seq=False))
        for e in extra:
            recs.append(_ul_rec(name, e, read_len, 0x800, seq=False))

    for t in tests:
        for side in ("pass", "fail"):
            pn, qn = ix["{}_{}_p".format(t, side)], ix["{}_{}_q".format(t, side)]
            junction(names[pn], names[qn], n=1)
            ok = side == "pass"
            prim = dict(ref=pn, pos=50000 - 12000, q=(100, 12100), rev=False)
            supp = dict(ref=qn, pos=0, q=(12150, 24150), rev=False)
            if t == "mapq":
                supp["mapq"] = 30 if ok else 29
            elif t == "len":
                m = 10000 if ok else 9999
                supp["q"] = (12150, 12150 + m)
            elif t == "dist":
                supp["pos"] = 100 if ok else 101
            elif t == "overlap":
                q0 = 6100 if ok else 6099
                supp["q"] = (q0, q0 + 12000)
            else:
                q0 = 22098 if ok else 22099
                supp["q"] = (q0, q0 + 12000)
            pair_read("t_{}_{}".format(t, side), prim, supp)
    # AS ties: two supplementaries with the same score, the first one counts
    for k, (t1, t2) in enumerate((("c", "S"), ("s", "I"), ("C", "i"))):
        prim = dict(ref=ix["tie_p"], pos=38000, q=(100, 12100), rev=False, AS=(5000, "I"))
        s1 = dict(ref=ix["tie_q"], pos=0, q=(12150, 24150), rev=False, AS=(100, t1))
        s2 = dict(ref=ix["tie_z"], pos=0, q=(12150, 24150), rev=False, AS=(100, t2))
        pair_read("tie{}".format(k), prim, s1, extra=(s2,))
    # a supplementary before its primary, one on the primary's own contig, and the supplementaries of a failed primary
    p = dict(ref=ix["h"], pos=38000, q=(100, 12100), rev=False)
    s = dict(ref=ix["i"], pos=0, q=(12150, 24150), rev=False)
    recs.append(_ul_rec("early", s, 24250, 0x800, seq=False))
    recs.append(_ul_rec("early", p, 24250))
    recs.append(_ul_rec("early", dict(p, pos=0), 24250, 0x800, seq=False))
    recs.append(_ul_rec("weak", dict(p, mapq=5), 24250))
    recs.append(_ul_rec("weak", s, 24250, 0x800, seq=False))
    recs.append(_ul_rec("weak", s, 24250, 0x800, seq=False))
    # flags that are neither primary nor supplementary, and an unmapped record
    recs.append(_ul_rec("early", s, 24250, 0x100, seq=False))
    recs.append(dict(_ul_rec("early", s, 24250, 0x4), ref=-1, pos=-1))
    recs.append(_ul_rec("dup", p, 24250, 0x400))
    return names, lengths, recs


def write_agp(asm: Assembly, path: str, gap: int = 100, prefix: str = "group") -> list:
    """The true layout of ``asm`` as an AGP: one scaffold per chromosome (``{prefix}{c + 1}``), its contigs in order, each
    W line oriented so that the contig reads along the chromosome ('-' for reverse-complemented ones), with a U gap of
    ``gap`` bp between neighbours.  Returns the W pieces (scaffold, scaffold start, contig id, orientation) in file order."""
    pieces = []
    with open(path, "w") as f:
        for c in range(asm.nchr):
            pos, part = 1, 1
            ids = np.nonzero(asm.chrom == c)[0]
            for k, i in enumerate(ids.tolist()):
                if k:
                    f.write("{}{}\t{}\t{}\t{}\tU\t{}\tscaffold\tyes\tproximity_ligation\n".format(
                        prefix, c + 1, pos, pos + gap - 1, part, gap))
                    pos += gap
                    part += 1
                ln = int(asm.lengths[i])
                ori = "-" if asm.ori[i] else "+"
                f.write("{}{}\t{}\t{}\t{}\tW\t{}\t1\t{}\t{}\n".format(prefix, c + 1, pos, pos + ln - 1, part, asm.names[i], ln, ori))
                pieces.append((c, pos, i, ori))
                pos += ln
                part += 1
    return pieces
