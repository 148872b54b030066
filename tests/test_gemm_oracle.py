"""Host checks of tests/gemm_oracle.py, the reference of the tensor-core pre-expansion: the exact product, the operand
encodings it emulates, the path choice it predicts, and that the 2e-6 bar of tests/test_gpu_gemm_scale.py fails for
every plausible defect of the GEMM on the inputs those tests use."""

import numpy as np
import pytest
import scipy.sparse as sp

from tests import gemm_oracle as go

# the correct encodings leave only their representation error (2^-22 per product and the fp32 reciprocal of the column
# sum); the GPU adds its fp32 accumulation on top, so the emulation must sit well inside the bar
ENCODING_SHARE = 0.25
# a defect must move the emulated product at least this many bars away
DEFECT_FACTOR = 10.0


@pytest.fixture(scope="module")
def kcut():
    link = go.kcut_matrix()
    cols = np.arange(*go.KCUT_SHARDS[1])
    return link, cols, go.exact_m1_cols(go.normalize(link), cols)


@pytest.fixture(scope="module")
def hub():
    link = go.hub_matrix(2 ** 23 - 1)
    cols = np.arange(2990, 3010)          # the hub (3001) and its neighbourhood
    return link, cols, go.exact_m1_cols(go.normalize(link), cols)


def test_exact_m1_cols_matches_dense_product():
    for n, seed in [(1, 0), (65, 1), (300, 2)]:
        link = go.random_counts(n, min(n, 40), 3000, seed)
        m0 = go.normalize(link)
        d = m0.toarray().astype(np.float64)
        full = d @ d
        for cols in (slice(None), np.array([0, n - 1]), np.arange(n)[::7]):
            got = go.exact_m1_cols(m0, cols)
            assert got.shape == full[:, cols].shape
            assert np.allclose(got, full[:, cols], rtol=1e-14, atol=0)
            assert np.array_equal(got != 0, full[:, cols] != 0)
        assert np.allclose(np.asarray(d.sum(axis=0)), 1.0, rtol=1e-6)


def test_normalize_is_fp32_of_fp64_quotient():
    link = go.random_counts(200, 30, 5000, 3)
    m0 = go.normalize(link)
    d = link.toarray().astype(np.float64)
    assert np.array_equal(m0.toarray(), (d / d.sum(axis=0)).astype(np.float32))


def test_split3_is_exact_bf16():
    rng = np.random.default_rng(4)
    x = np.concatenate([rng.random(10000).astype(np.float32), rng.integers(0, 65536, 1000).astype(np.float32),
                        np.float32([1e-30, 3.0e38, 2.0 ** -23, 1.0])])
    h = go.split3(x)
    assert np.array_equal(h[0] + h[1] + h[2], x.astype(np.float64))
    for p in h:
        assert not np.any(p.astype(np.float32).view(np.uint32) & 0xFFFF)      # each part is a bf16 value


@pytest.mark.parametrize("case", ["kcut", "hub", "clip", "weights"])
def test_encodings_reproduce_the_operands(case, kcut, hub):
    link = {"kcut": lambda: kcut[0], "hub": lambda: hub[0], "clip": lambda: go.planted_count(5000),
            "weights": lambda: go.planted_count(100003)}[case]()
    if case == "kcut":
        link = link[:, :3000]          # the columns suffice: every column is encoded on its own
        link = sp.csc_matrix(link)
    s = go.colsums(link)
    col = np.repeat(np.arange(link.shape[1]), np.diff(link.indptr))
    x32 = lambda clip: (np.minimum(link.data, np.float32(clip)).astype(np.float64) / s[col]).astype(np.float32)
    encs = ["weights"] if case == "weights" else ["f16", "bf16"]
    for enc in encs:
        A, B, passes, e = go.encode(link, enc)
        e = np.asarray(e)
        if enc == "f16":
            # one f16 count plane: min(C, 2048) * 2^-e_k exactly; hi + lo within 2^-22 of fp32(min(C, 2048) / s) * 2^e_k
            assert len(A) == 1 and len(B) == 2 and passes == go.PASSES_F16
            assert np.array_equal(np.ldexp(A[0].data, e), np.minimum(link.data, 2048.0))
            b = np.ldexp(B[0].data + B[1].data, -e)
            x = x32(go.F16_CLIP).astype(np.float64)
            assert (np.abs(b - x) / x).max() <= 2.0 ** -22
            for p in A + B:
                assert np.array_equal(p.data.astype(np.float16).astype(np.float64), p.data)
            if case == "hub":
                # the hub's count-1 entries are the f16 subnormal 2^-23
                hub_col = A[0][:, 3001].toarray().ravel()
                assert (hub_col == 2.0 ** -23).sum() == 2 ** 23 - 1 - 4095 * 2048
        elif enc == "bf16":
            assert len(A) == 1 and len(B) == 3 and passes == go.PASSES_1
            assert np.array_equal(A[0].data, np.minimum(link.data, 256.0))
            assert np.array_equal(B[0].data + B[1].data + B[2].data, x32(go.BF16_CLIP).astype(np.float64))
        else:
            assert len(A) == 3 and len(B) == 3 and passes == go.PASSES_3
            assert np.array_equal(A[0].data + A[1].data + A[2].data, link.data.astype(np.float64))
            assert np.array_equal(B[0].data + B[1].data + B[2].data, x32(3.0e38).astype(np.float64))


def test_expected_preexp_thresholds():
    e = go.expected_preexp
    hub_lo, hub_hi = go.hub_matrix(2 ** 23 - 1), go.hub_matrix(2 ** 23)
    assert go.colsums(hub_lo).max() == 2 ** 23 - 1 and go.colsums(hub_hi).max() == 2 ** 23
    assert (e(hub_lo)["fmt_a"], e(hub_lo)["passes"], e(hub_lo)["clipped"]) == (go.F16, 2, False)
    assert (e(hub_hi)["fmt_a"], e(hub_hi)["b_planes"], e(hub_hi)["passes"], e(hub_hi)["clipped"]) == (go.BF16, 3, 3, True)
    for v, fmt, clipped in [(2048, None, False), (2049, None, True), (256, "bf16", False), (257, "bf16", True),
                            (2048, "bf16", True)]:
        p = e(go.planted_count(v), fmt)
        assert p["clipped"] == clipped and p["a_planes"] == 1, (v, fmt)
    for v in (65535, 65536, 65537, 100003):
        p = e(go.planted_count(v))
        assert p["weights"] == (v >= 65536) and p["a_planes"] == (3 if v >= 65536 else 1), v
        assert p["passes"] == (6 if v >= 65536 else 2) and p["clipped"] == (v < 65536), v
    w = sp.csc_matrix(go.planted_count(3).astype(np.float32) * np.float32(0.5))
    assert e(w)["weights"]
    # K cuts: the budget of 16 GB of planes per chunk, the HH_GEMM_KCHUNKS setting and its clamp to 64-wide chunks
    n = go.KCUT_N
    fake = sp.identity(n, dtype=np.float32, format="csc")
    assert (e(fake)["k_chunks"], e(fake)["kw"], e(fake)["segments"]) == (2, 30016, 1)
    assert (e(fake, kchunks=1)["k_chunks"], e(fake, kchunks=1)["kw"], e(fake, kchunks=1)["segments"]) == (1, 60032, 2)
    assert (e(fake, kchunks=7)["k_chunks"], e(fake, kchunks=7)["kw"]) == (7, 8576)
    c3 = sp.identity(50000, dtype=np.float32, format="csc")
    assert (e(c3)["k_chunks"], e(c3)["segments"]) == (1, 2)
    assert e(c3, "bf16")["k_chunks"] == 2
    small = sp.identity(1100, dtype=np.float32, format="csc")
    assert (e(small, kchunks=17)["k_chunks"], e(small, kchunks=17)["kw"]) == (9, 128)
    assert (e(small, kchunks=1000)["k_chunks"], e(small, kchunks=1000)["kw"]) == (18, 64)


def test_correct_emulation_is_inside_the_bar(kcut, hub):
    link, cols, exact = kcut
    for enc in ("f16", "bf16"):
        same, err = go.rel_error(go.emulate_m1_cols(link, cols, enc), exact)
        assert same and err <= ENCODING_SHARE * go.BAR, (enc, err)
    link, cols, exact = hub
    for enc in ("f16", "bf16"):
        same, err = go.rel_error(go.emulate_m1_cols(link, cols, enc), exact)
        assert same and err <= ENCODING_SHARE * go.BAR, (enc, err)
    for v, enc in [(2049, "f16"), (257, "bf16"), (65535, "f16"), (100003, "weights")]:
        link = go.planted_count(v)
        same, err = go.rel_error(go.emulate_m1_cols(link, slice(None), enc), go.exact_m1_cols(go.normalize(link), slice(None)))
        assert same and err <= ENCODING_SHARE * go.BAR, (v, enc, err)


def _defect(link, cols, exact, enc="f16", **kw):
    same, err = go.rel_error(go.emulate_m1_cols(link, cols, enc, **kw), exact)
    return err if same else np.inf


def test_bar_catches_flushed_subnormals(kcut, hub):
    # the hub's count-1 entries (2^-23) and the f16 lo planes below 2^-14
    assert _defect(*hub, flush_subnormals=True) >= DEFECT_FACTOR * go.BAR
    assert _defect(*kcut, flush_subnormals=True) >= DEFECT_FACTOR * go.BAR


def test_bar_catches_a_dropped_lo_plane(kcut):
    assert _defect(*kcut, drop_lo=True) >= DEFECT_FACTOR * go.BAR


def test_bar_catches_an_exponent_off_by_one(kcut, hub):
    # 2^e_k cancels only if both operands use the same e_k
    assert _defect(*kcut, e_off_a=1) >= DEFECT_FACTOR * go.BAR
    assert _defect(*hub, e_off_a=-1) >= DEFECT_FACTOR * go.BAR


@pytest.mark.parametrize("kchunks,which", [(1, 1), (None, 1), (7, 3)])
def test_bar_catches_a_lost_k_range(kcut, kchunks, which):
    """a densify segment (HH_GEMM_KCHUNKS=1: the second, partial segment) or a K chunk (default: two chunks; 7 chunks)
    left out of the sum"""
    link, cols, exact = kcut
    p = go.expected_preexp(link, kchunks=kchunks)
    if kchunks == 1:
        assert p["k_chunks"] == 1 and p["segments"] == 2
        lo, hi = go.HG_SEG, p["kw"]
    else:
        assert p["k_chunks"] == (2 if kchunks is None else 7)
        lo, hi = which * p["kw"], min(go.KCUT_N, (which + 1) * p["kw"])
    assert _defect(link, cols, exact, drop_k=(lo, hi)) >= DEFECT_FACTOR * go.BAR


@pytest.mark.parametrize("v,enc", [(2049, "f16"), (257, "bf16"), (65535, "f16")])
def test_bar_catches_a_missing_clip_correction(v, enc):
    link = go.planted_count(v)
    exact = go.exact_m1_cols(go.normalize(link), slice(None))
    assert _defect(link, slice(None), exact, enc, clip_fix=False) >= DEFECT_FACTOR * go.BAR
    assert _defect(link, slice(None), exact, enc) <= ENCODING_SHARE * go.BAR
