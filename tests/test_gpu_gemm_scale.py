"""GPU checks of the tensor-core pre-expansion M1 = M0 . M0 (hh_k_gemm_densify + hh_k_syrk + hh_k_clip_fix, through
hh_mcl_create_ex) at the benchmark's size and at the boundaries of its operand encodings.

Every case asserts through Mcl.preexp the path it targets (engine, operand formats, planes, passes, K chunks, whether the
clip correction ran), as tests/gemm_oracle.expected_preexp predicts it from the matrix, and then holds every stored entry of
M1 to an identical non-zero pattern and 2e-6 relative of the exact fp64 product of the device's own M0 (Mcl.m0(), which
other tests hold bit-exact): the test is about the GEMM alone.  The three inputs DESIGN.md section 2 names as exceeding 2e-6
by accumulation are held to its 5e-6 accumulation band instead.

  C3 (bench.py's matrix: 50k contigs, 200M pairs, seed 12345), every entry: the default path (scaled f16, one K chunk of
     two densify segments), HH_GEMM_FMT=bf16 (two K chunks) and the --normalize_by_nlinks matrix (three planes each side,
     six passes, two K chunks).  The reference is a dense fp64 GEMM on the device (cuBLAS DGEMM, error ~1e-14), spot-checked
     against SciPy's fp64 sparse product on the host; M1 is fetched in blocks of columns.
  C3 column shards with bounds that are not tile-aligned, one straddling column 32,768: bit-identical to the whole run.
  K cuts at n = 60,000: the default cut (two chunks), one chunk (two densify segments, the second partial) and seven.
  Encoding boundaries: a column sum of 2^23 - 1 (f16 with subnormal 2^-23 operands) and 2^23 (exact bf16), the clip
     thresholds 2048 / 256 and one above, counts 65,535 .. 100,003 (the three-plane weights path from 65,536 on).
  Ragged shapes n = 1 .. 257 and the clamp of HH_GEMM_KCHUNKS to 64-wide chunks.

Run with -s to see, per case, the worst error as a fraction of the bar and the device memory in use."""

import json
import time

import numpy as np
import pytest
import torch

from tests import gemm_oracle as go

pytestmark = pytest.mark.gpu

BAR = go.BAR
N_CONTIGS, N_CHR, MEAN_LEN, N_PAIRS, SEED = 50000, 24, 20000, 200_000_000, 12345
BAND = go.ACCUMULATION_BAND
BLOCK = 2048                    # columns of M1 compared at a time at C3
PEAK = {"bytes": 0}


def sample_memory():
    free, total = torch.cuda.mem_get_info(0)
    PEAK["bytes"] = max(PEAK["bytes"], total - free)


def report(case, **kw):
    sample_memory()
    kw["device_gb_in_use_peak"] = round(PEAK["bytes"] / 1e9, 2)
    print("\ngemm-scale {} {}".format(case, json.dumps(kw)))


def set_fmt(monkeypatch, fmt):
    if fmt is None:
        monkeypatch.delenv("HH_GEMM_FMT", raising=False)
    else:
        monkeypatch.setenv("HH_GEMM_FMT", fmt)


def set_kchunks(monkeypatch, kchunks):
    if kchunks is None:
        monkeypatch.delenv("HH_GEMM_KCHUNKS", raising=False)
    else:
        monkeypatch.setenv("HH_GEMM_KCHUNKS", str(kchunks))


def assert_path(mc, want, **explicit):
    """mc.preexp is the path expected_preexp predicts, and the values this case targets."""
    p = mc.preexp
    assert p["mode"] == "dense"
    for k in ("fmt_a", "fmt_b", "a_planes", "b_planes", "passes", "k_chunks", "chunk_kb"):
        if k not in explicit:
            assert p[k] == want[k], (k, p[k], want[k])
    assert p["clip"] == np.float32(want["clip"])
    assert (p["clip_ms"] > 0) == want["clipped"], (p["clip_ms"], want["clipped"])
    for k, v in explicit.items():
        if k == "clipped":
            assert (p["clip_ms"] > 0) == v
        elif k == "segments":
            assert want["segments"] == v and p["k_chunks"] == want["k_chunks"]
        else:
            assert p[k] == v, (k, p[k], v)


@pytest.fixture(scope="module")
def ctx():
    from haphic_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def check_whole(ctx, link, fmt=None, kchunks=None, bar=BAR, **explicit):
    """Mcl(preexp="dense") of a small matrix: path, pattern and every entry against the exact product.  Returns M1 and the
    worst error as a fraction of the 2e-6 bar."""
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    mat = LinkMatrix.from_csc(ctx, link)
    mc = Mcl(mat, preexp="dense")
    try:
        assert_path(mc, go.expected_preexp(link, fmt, kchunks), **explicit)
        got = mc.m1()
        same, err = go.rel_error(got, go.exact_m1_cols(mc.m0(), slice(None)))
        assert same, "non-zero pattern differs"
        assert err <= bar, err
        return got, err / BAR
    finally:
        mc.close()
        mat.close()


# ---------------------------------------------------------------------------------------------------------------------------
# ragged shapes and the K-chunk clamp
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [None, "bf16"])
@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 127, 128, 129, 255, 257])
def test_ragged_shapes(ctx, monkeypatch, n, fmt):
    set_fmt(monkeypatch, fmt)
    link = go.random_counts(n, max(1, n // 2), 300, seed=n)
    got, frac = check_whole(ctx, link, fmt, fmt_a=go.BF16 if fmt else go.F16, k_chunks=1)
    if n == 1:
        assert got.shape == (1, 1) and got[0, 0] == np.float32(1.0)
    report("ragged n={} fmt={}".format(n, fmt or "default"), worst_over_bar=frac)


@pytest.mark.parametrize("kchunks,chunks", [(17, 9), (1000, 18)])
def test_kchunk_clamp(ctx, monkeypatch, kchunks, chunks):
    """HH_GEMM_KCHUNKS above n / 64: chunks of 128 columns (17) or of one k-block (1000, the last chunk 12 columns wide)"""
    set_fmt(monkeypatch, None)
    set_kchunks(monkeypatch, kchunks)
    n = 1100
    link = go.random_counts(n, 400, 3000, seed=21)
    want = go.expected_preexp(link, None, kchunks)
    assert want["k_chunks"] == -(-n // want["kw"]) == chunks
    _got, frac = check_whole(ctx, link, None, kchunks, k_chunks=chunks)
    report("kchunks={} n={}".format(kchunks, n), worst_over_bar=frac, kw=want["kw"])


# ---------------------------------------------------------------------------------------------------------------------------
# encoding boundaries
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hub_sum,fmt", [(2 ** 23 - 1, None), (2 ** 23 - 1, "bf16"), (2 ** 23, None), (2 ** 23, "bf16")])
def test_column_sum_boundary(ctx, monkeypatch, hub_sum, fmt):
    """a hub column of sum 2^23 - 1 keeps the scaled f16 encoding with e_k = 23, so its count-1 entries enter the count
    plane as the f16 subnormal 2^-23; a sum of 2^23 switches to the exact bf16 encoding (which clips the 2048s at 256).
    Two of these inputs exceed 2e-6 by accumulation, not by encoding (DESIGN.md section 2): the default f16 drain period of
    three k-blocks (4.84e-6, and 3.8e-7 with a drain every two k-blocks), and the fp32 clip correction of 4,095 clipped
    counts in one column (2.04e-6); they are held to the accumulation band."""
    set_fmt(monkeypatch, fmt)
    monkeypatch.delenv("HH_GEMM_CHUNK", raising=False)
    link = go.hub_matrix(hub_sum)
    s = go.colsums(link)
    assert s.max() == s[3001] == hub_sum and go.exponent(s)[3001] == (23 if hub_sum < 2 ** 23 else 24)
    f16 = fmt is None and hub_sum < 2 ** 23
    path = dict(fmt_a=go.F16 if f16 else go.BF16, b_planes=2 if f16 else 3, passes=2 if f16 else 3, clipped=not f16)
    band = BAR if (fmt == "bf16" and hub_sum < 2 ** 23) else BAND
    _got, frac = check_whole(ctx, link, fmt, bar=band, **path)
    kw = {}
    if f16:
        # the same planes drained every two k-blocks: inside the 2e-6 bar, so the subnormal operands multiply exactly
        monkeypatch.setenv("HH_GEMM_CHUNK", "2")
        _got, kw["worst_over_bar_drain_2"] = check_whole(ctx, link, fmt, chunk_kb=2, **path)
    report("colsum={} fmt={}".format(hub_sum, fmt or "default"), worst_over_bar=frac, **kw)


@pytest.mark.parametrize("value,fmt,clipped", [(2048, None, False), (2049, None, True), (256, "bf16", False), (257, "bf16", True)])
def test_clip_threshold(ctx, monkeypatch, value, fmt, clipped):
    """a count equal to the clip threshold enters the GEMM whole; one above it is clipped and finished by hh_k_clip_fix"""
    set_fmt(monkeypatch, fmt)
    link = go.planted_count(value)
    _got, frac = check_whole(ctx, link, fmt, fmt_a=go.BF16 if fmt else go.F16, a_planes=1, clipped=clipped)
    report("max count={} fmt={}".format(value, fmt or "default"), worst_over_bar=frac)


@pytest.mark.parametrize("value", [65535, 65536, 65537, 100003])
def test_large_counts(ctx, monkeypatch, value):
    """counts of 65,536 and more leave the integer encodings: three bf16 planes each side, six passes, no clip"""
    set_fmt(monkeypatch, None)
    link = go.planted_count(value)
    if value < 65536:
        explicit = dict(fmt_a=go.F16, a_planes=1, passes=2, clipped=True)
    else:
        explicit = dict(fmt_a=go.BF16, a_planes=3, b_planes=3, passes=6, clipped=False)
    _got, frac = check_whole(ctx, link, None, **explicit)
    report("max count={}".format(value), worst_over_bar=frac)


# ---------------------------------------------------------------------------------------------------------------------------
# K cuts at size (column shards only: the GEMM work stays small, the operand planes are full size)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kcut_link():
    return go.kcut_matrix()


@pytest.mark.parametrize("kchunks,chunks,segments", [(None, 2, 1), (1, 1, 2), (7, 7, 1)])
def test_k_cuts_at_size(monkeypatch, kcut_link, kchunks, chunks, segments):
    from haphic_b200._lib import Context
    from haphic_b200.links import LinkMatrix
    from haphic_b200.mcl import Mcl
    set_fmt(monkeypatch, None)
    set_kchunks(monkeypatch, kchunks)
    t0 = time.perf_counter()
    want = go.expected_preexp(kcut_link, None, kchunks)
    worst = 0.0
    c = Context(0)
    try:
        mat = LinkMatrix.from_csc(c, kcut_link)
        m0 = None
        for lo, hi in go.KCUT_SHARDS:
            mc = Mcl(mat, col_lo=lo, col_hi=hi, preexp="dense")
            assert_path(mc, want, fmt_a=go.F16, k_chunks=chunks, segments=segments, clipped=False)
            if m0 is None:
                m0 = mc.m0()
            got = mc.m1()
            sample_memory()
            mc.close()
            same, err = go.rel_error(got, go.exact_m1_cols(m0, np.arange(lo, hi)))
            assert same, (lo, hi)
            assert err <= BAR, (lo, hi, err)
            worst = max(worst, err / BAR)
        mat.close()
    finally:
        c.close()
    report("kcut n={} kchunks={}".format(go.KCUT_N, kchunks or "default"), worst_over_bar=worst, kw=want["kw"],
           seconds=round(time.perf_counter() - t0, 1))


# ---------------------------------------------------------------------------------------------------------------------------
# C3: the benchmark's matrix, every entry
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def c3():
    from haphic_b200 import synth
    from haphic_b200._lib import Context
    from haphic_b200.links import LinkTable, name_rank
    c = Context(0)
    asm = synth.make_assembly(N_CHR, N_CONTIGS, MEAN_LEN, seed=SEED)
    rank = name_rank(asm.names)
    in_nx = np.ones(asm.n, np.uint8)
    rec = synth.make_pairs_range(asm, 0, N_PAIRS, seed=SEED + 1, device="cuda")
    tab = LinkTable(c, asm.lengths, rank, in_nx, 500000, capacity_hint=int(0.45 * N_PAIRS))
    tab.add(rec, asynchronous=True)
    tab.finish()
    del rec
    keep = np.ones(asm.n, np.uint8)
    mats = {}
    for name, norm in (("counts", False), ("nlinks", True)):
        index, _ = tab.linked_index(keep, normalize_by_nlinks=norm)
        tail = np.nonzero(index < 0)[0].astype(np.int32)
        mats[name] = tab.to_matrix(keep, tail, normalize_by_nlinks=norm)
    tab.close()
    torch.cuda.empty_cache()
    yield {"ctx": c, "mats": mats, "scipy_fp32": {}}
    for m in mats.values():
        m.close()
    c.close()


def dense_fp64(m0, dev):
    """M0 as a dense fp64 [n, n] tensor on the device (20 GB at n = 50k)."""
    n = m0.shape[0]
    rows = torch.from_numpy(m0.indices.astype(np.int64)).to(dev)
    cols = torch.repeat_interleave(torch.arange(n, device=dev), torch.from_numpy(np.diff(m0.indptr)).to(dev))
    d = torch.zeros((n, n), dtype=torch.float64, device=dev)
    d[rows, cols] = torch.from_numpy(m0.data).to(dev).double()
    del rows, cols
    return d


def fetch_block(mc, lo, hi, pinned):
    """M1[:, lo:hi] into the pinned host buffer (column-major: row j of the buffer is column lo + j)."""
    from haphic_b200._lib import check, load, ptr
    view = pinned[: hi - lo]
    check(load().hh_mcl_fetch_m1_cols(mc._h, int(lo), int(hi), ptr(view)))
    return view


@pytest.mark.parametrize("case", ["auto", "bf16", "nlinks"])
def test_c3_every_entry(c3, monkeypatch, case):
    from haphic_b200.mcl import Mcl
    fmt = "bf16" if case == "bf16" else None
    set_fmt(monkeypatch, fmt)
    set_kchunks(monkeypatch, None)
    mat = c3["mats"]["nlinks" if case == "nlinks" else "counts"]
    n = mat.n
    t0 = time.perf_counter()
    want = go.expected_preexp(mat.to_scipy(), fmt)
    mc = Mcl(mat)                                   # the engine `auto` picks, as bench.py
    dev = torch.device("cuda", 0)
    m0d = None
    try:
        if case == "auto":
            assert_path(mc, want, fmt_a=go.F16, a_planes=1, b_planes=2, passes=2, k_chunks=1, segments=2)
        elif case == "bf16":
            assert_path(mc, want, fmt_a=go.BF16, a_planes=1, b_planes=3, passes=3, k_chunks=2, segments=1)
        else:
            assert_path(mc, want, fmt_a=go.BF16, a_planes=3, b_planes=3, passes=6, k_chunks=2, clipped=False)
        gemm = {k: mc.preexp[k] for k in ("densify_ms", "gemm_ms", "clip_ms")}
        m0 = mc.m0()
        m0d = dense_fp64(m0, dev)
        pinned = torch.empty((BLOCK, n), dtype=torch.float32, pin_memory=True)
        worst, where, nnz = 0.0, None, 0
        for lo in range(0, n, BLOCK):
            hi = min(n, lo + BLOCK)
            ref = m0d @ m0d[:, lo:hi]                                       # [n, hi - lo]
            got = fetch_block(mc, lo, hi, pinned).to(dev).T.double()
            sample_memory()
            nz = ref != 0
            assert torch.equal(got != 0, nz), "non-zero pattern differs in columns [{}, {})".format(lo, hi)
            rel = torch.where(nz, (got - ref).abs() / torch.where(nz, ref, 1.0), 0.0)
            k = int(rel.argmax())
            if float(rel.view(-1)[k]) > worst:
                worst, where = float(rel.view(-1)[k]), (k // (hi - lo), lo + k % (hi - lo))
            nnz += int(nz.sum())
            del ref, got, nz, rel
        # the device reference against SciPy's fp64 product on the host, a few columns (tile and segment edges)
        rng = np.random.default_rng(7)
        spot = np.unique(np.concatenate([[0, 127, 128, 32767, 32768, n - 1], rng.integers(0, n, 4)]))
        host = go.exact_m1_cols(m0, spot)
        devref = (m0d @ m0d[:, torch.from_numpy(spot).to(dev)]).cpu().numpy()
        same, err_ref = go.rel_error(devref, host)
        assert same and err_ref <= 1e-12, err_ref
        # context, not asserted: SciPy's fp32 product (the reference's own arithmetic) on 200 of the same columns
        key = "nlinks" if case == "nlinks" else "counts"
        if key not in c3["scipy_fp32"]:
            sc_cols = np.sort(rng.choice(n, 200, replace=False))
            sc = (m0 @ m0[:, sc_cols]).toarray()
            ex = (m0d @ m0d[:, torch.from_numpy(sc_cols).to(dev)]).cpu().numpy()
            c3["scipy_fp32"][key] = go.rel_error(sc, ex)[1] / BAR
        # the weights encoding (six passes) is held to the accumulation band at this size (DESIGN.md section 2)
        assert worst <= (BAND if case == "nlinks" else BAR), (worst, where)
        report("C3 {}".format(case), worst_over_bar=round(worst / BAR, 4), worst_at=where, stored_entries=nnz,
               spot_check_ref_err=err_ref, scipy_fp32_worst_over_bar_200cols=round(c3["scipy_fp32"][key], 4),
               preexp_ms=gemm, k_chunks=mc.preexp["k_chunks"], passes=mc.preexp["passes"],
               seconds=round(time.perf_counter() - t0, 1))
    finally:
        mc.close()
        del m0d
        torch.cuda.empty_cache()


def test_c3_shards_bit_identical(c3, monkeypatch):
    """column shards whose bounds are not tile-aligned, one straddling column 32,768 (the second densify segment), and
    the first and last 100 columns: bit-identical to the whole run's columns"""
    from haphic_b200.mcl import Mcl
    set_fmt(monkeypatch, None)
    set_kchunks(monkeypatch, None)
    mat = c3["mats"]["counts"]
    n = mat.n
    ranges = [(32700, 32900), (0, 100), (n - 100, n)]
    whole = Mcl(mat, preexp="dense")
    path = {k: whole.preexp[k] for k in ("mode", "fmt_a", "passes", "k_chunks")}
    assert path == {"mode": "dense", "fmt_a": go.F16, "passes": 2, "k_chunks": 1}
    want = {r: whole.m1(*r) for r in ranges}
    whole.close()
    for lo, hi in ranges:
        part = Mcl(mat, col_lo=lo, col_hi=hi, preexp="dense")
        assert {k: part.preexp[k] for k in path} == path
        got = part.m1()
        sample_memory()
        part.close()
        assert got.shape == (n, hi - lo)
        assert np.array_equal(got, want[(lo, hi)]), (lo, hi)
    report("C3 shards", ranges=ranges)
