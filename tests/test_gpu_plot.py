"""`haphic plot` on the device against the reference's goldens (tests/golden/make_plot_golden.py) and against torch /
numpy reconstructions at larger sizes."""

import ast
import gzip
import logging
import os
import pickle
import shutil

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from haphic_b200 import hicio, plot, synth  # noqa: E402
from haphic_b200._lib import Context  # noqa: E402
from tests import plot_oracle  # noqa: E402

GOLD = ("main", "specified", "allkept")


@pytest.fixture(scope="module")
def ctx():
    c = Context(0)
    yield c
    c.close()


def golden(golden_dir, tag):
    return np.load(os.path.join(golden_dir, "plot_{}.npz".format(tag)))


def case_files(z, d):
    agp, pairs = os.path.join(d, "asm.agp"), os.path.join(d, "aln.pairs")
    with open(agp, "w") as f:
        f.write(str(z["agp"]))
    with open(pairs, "w") as f:
        f.write(str(z["pairs"]))
    return agp, pairs


def layout_of(z, agp):
    return plot.Layout(agp, int(z["bin_size"]) * 1000, int(z["min_len"]), str(z["specified"]) or None)


def records_of(layout, pairs):
    return np.concatenate(list(hicio.pairs_batches(pairs, "pairs", layout.name_index(), bed_path=None, inter_only=False)))


def count(ctx, layout, batches, asynchronous=False):
    cm = plot.ContactMap(ctx, layout)
    for b in batches:
        cm.add(b, asynchronous=asynchronous)
    assert cm.error() is None
    cm.finish()
    m = cm.fetch()
    cm.close()
    return m


@pytest.mark.parametrize("tag", GOLD)
def test_matrix_is_bit_exact_for_pairs_gz_and_bam(ctx, golden_dir, tmp_path, tag):
    z = golden(golden_dir, tag)
    agp, pairs = case_files(z, str(tmp_path))
    L = layout_of(z, agp)
    rec = records_of(L, pairs)
    m = count(ctx, L, [rec])
    assert m.dtype == np.int64 and np.array_equal(m, z["matrix"])
    gz = str(tmp_path / "aln.pairs.gz")
    with open(pairs, "rb") as fi, gzip.open(gz, "wb") as fo:
        shutil.copyfileobj(fi, fo)
    rec_gz = np.concatenate(list(hicio.pairs_batches(gz, "bgzipped_pairs", L.name_index(), bed_path=None, inter_only=False)))
    assert np.array_equal(count(ctx, L, [rec_gz]), z["matrix"])
    # BAM: records whose names are missing from the AGP cannot be written with a reference id; they are skipped anyway
    keep = (rec[:, 0] >= 0) & (rec[:, 2] >= 0)
    bam = str(tmp_path / "aln.bam")
    hicio.write_bam(bam, L.names, [10 ** 7] * len(L.names), rec[keep])
    rec_bam = np.concatenate(list(hicio.bam_batches(bam, L.name_index(), inter_only=False)))
    assert np.array_equal(count(ctx, L, [rec_bam]), z["matrix"])


def test_error_is_the_first_offending_record(ctx, golden_dir, tmp_path, monkeypatch):
    z = golden(golden_dir, "error")
    agp, pairs = case_files(z, str(tmp_path))
    monkeypatch.chdir(tmp_path)
    args = plot.parse_arguments([agp, pairs, "--bin_size", "100"])
    with pytest.raises(Exception) as e:
        plot.run(args, ctx=ctx)
    assert str(e.value) == str(z["error"])


def test_batches_async_and_device_records_equal_one_batch(ctx, golden_dir, tmp_path):
    z = golden(golden_dir, "main")
    agp, pairs = case_files(z, str(tmp_path))
    L = layout_of(z, agp)
    rec = records_of(L, pairs)
    one = count(ctx, L, [rec])
    assert np.array_equal(count(ctx, L, np.array_split(rec, 37)), one)
    dev = torch.from_numpy(rec).cuda()
    assert np.array_equal(count(ctx, L, [dev]), one)
    parts = [p.contiguous() for p in torch.tensor_split(dev, 11)]
    assert np.array_equal(count(ctx, L, parts, asynchronous=True), one)
    assert np.array_equal(count(ctx, L, [torch.from_numpy(rec)]), one)


def one_scaffold(tmp_path, length, bin_kb):
    agp = str(tmp_path / "one.agp")
    with open(agp, "w") as f:
        f.write("s1\t1\t{0}\t1\tW\tc\t1\t{0}\t+\n".format(length))
    return plot.Layout(agp, bin_kb * 1000, 0)


def test_skewed_streams_are_exact(ctx, tmp_path):
    L = one_scaffold(tmp_path, 200_000_000, 100)        # 2001 bins
    nb = L.nb
    g = torch.Generator(device="cuda")
    g.manual_seed(11)
    n_hot = (1 << 24) + 12345
    hot = torch.tensor([[0, 5_000_000, 0, 5_000_100]], dtype=torch.int32, device="cuda").repeat(n_hot, 1)
    m = 8_000_000
    pa = torch.randint(0, 200_000_000, (m,), generator=g, device="cuda", dtype=torch.int64)
    pb = (pa + torch.randint(-150_000, 150_000, (m,), generator=g, device="cuda")).clamp(0, 200_000_000 - 1)
    diag = torch.stack([torch.zeros_like(pa), pa, torch.zeros_like(pa), pb], 1).to(torch.int32)
    rec = torch.cat([hot, diag]).contiguous()
    cm = plot.ContactMap(ctx, L)
    cm.add(rec)
    cm.finish()
    got = torch.from_numpy(cm.fetch()).cuda()
    cm.close()
    ba, bb = rec[:, 1].long() // 100_000, rec[:, 3].long() // 100_000
    c = torch.bincount(ba * nb + bb, minlength=nb * nb).view(nb, nb)
    want = c + c.T - torch.diag(torch.diagonal(c))
    assert torch.equal(got, want)
    assert int(got[50, 50]) >= (1 << 24)


def c3_records(asm, n, seed):
    return synth.make_pairs(asm, n, seed=seed, device="cuda")


def test_c3_shape_at_500kb_matches_torch(ctx, tmp_path):
    asm = synth.make_assembly(nchr=24, n_contigs=50_000, mean_len=60_000, seed=31)
    agp = str(tmp_path / "c3.agp")
    pieces = synth.write_agp(asm, agp)
    L = plot.Layout(agp, 500_000, 1)
    rec = c3_records(asm, 200_000_000, 32)
    cm = plot.ContactMap(ctx, L)
    cm.add(rec, asynchronous=True)
    cm.finish()
    got = torch.from_numpy(cm.fetch()).cuda()
    cm.close()
    # the true layout: scaffold start of each contig and its orientation, bins of the scaffold coordinate
    start = np.zeros(asm.n, np.int64)
    rev = np.zeros(asm.n, bool)
    for _c, pos, i, ori in pieces:
        start[i], rev[i] = pos, ori == "-"
    goff, o = np.zeros(asm.nchr, np.int64), 0
    for c, g in enumerate(L.group_list):
        goff[c] = o
        o += L.group_size[g] // 500_000 + 1
    start_t, rev_t = torch.from_numpy(start).cuda(), torch.from_numpy(rev).cuda()
    len_t, goff_t = torch.from_numpy(asm.lengths).cuda(), torch.from_numpy(goff[asm.chrom]).cuda()

    def tbin(ids, pos):
        ids, raw = ids.long(), pos.long() + 1
        gpos = torch.where(rev_t[ids], start_t[ids] + len_t[ids] - raw, start_t[ids] + raw - 1)
        return goff_t[ids] + (gpos - 1) // 500_000

    nb = L.nb
    c = torch.zeros(nb * nb, dtype=torch.int64, device="cuda")
    for part in torch.split(rec, 1 << 25):
        c += torch.bincount(tbin(part[:, 0], part[:, 1]) * nb + tbin(part[:, 2], part[:, 3]), minlength=nb * nb)
    c = c.view(nb, nb)
    want = c + c.T - torch.diag(torch.diagonal(c))
    assert torch.equal(got, want)


def test_kr_matches_golden_x_and_steps(ctx, golden_dir):
    z = np.load(os.path.join(golden_dir, "plot_bnewt.npz"))
    for name in z["names"]:
        A = z["A_" + name]
        counts = np.rint(A - 0.00001).astype(np.int64)
        assert np.array_equal(counts + 0.00001, A)
        (x, outer, inner, ok), = plot.kr_balance(counts, ctx=ctx)
        assert ok and [outer, inner] == z["steps_" + name].tolist(), name
        np.testing.assert_allclose(x, z["x_" + name], rtol=1e-10, atol=0, err_msg=name)


def test_kr_blocks_together_equal_one_by_one(ctx, golden_dir, tmp_path):
    z = golden(golden_dir, "allkept")
    L = layout_of(z, case_files(z, str(tmp_path))[0])
    blocks = L.blocks() + [(0, L.nb)]
    together = plot.kr_balance(z["matrix"], blocks, ctx=ctx)
    for blk, t in zip(blocks, together):
        (x, outer, inner, ok), = plot.kr_balance(z["matrix"], [blk], ctx=ctx)
        assert ok and (outer, inner) == t[1:3] and np.array_equal(x, t[0])


def test_kr_reports_non_convergence(ctx, golden_dir):
    z = golden(golden_dir, "main")
    (_x, outer, _inner, ok), = plot.kr_balance(z["matrix"], max_outer=1, ctx=ctx)
    assert not ok and outer == 1


def ulp_diff(a, b):
    return np.abs(a.view(np.int64) - b.view(np.int64))


@pytest.mark.parametrize("tag", GOLD)
def test_normalised_matrices_and_vmax(ctx, golden_dir, tmp_path, tag):
    z = golden(golden_dir, tag)
    L = layout_of(z, case_files(z, str(tmp_path))[0])
    cm = plot.ContactMap(ctx, counts=z["matrix"])
    try:
        for norm in ("KR", "log10", "none"):
            m, vmax = plot.normalize_matrix(cm, L, norm, 4.0, -1, raw=z["matrix"])
            wv = float(z["vmax_" + norm])
            if norm == "KR":
                want = z["norm_KR"]
                np.testing.assert_allclose(m, want, rtol=1e-9, atol=0)
                assert abs(vmax - wv) <= 1e-9 * abs(wv)
            elif norm == "log10":
                assert ulp_diff(m, z["norm_log10"]).max() <= 2
                assert abs(vmax - wv) <= 4 * np.spacing(wv)
            else:
                assert np.array_equal(m, z["matrix"]) and vmax == wv
    finally:
        cm.close()


class Lines(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def vmax_lines(lines):
    return [ln for ln in lines if "vmax" in ln or "Normaliz" in ln]


def test_run_writes_the_reference_pickle_and_a_pkl_input_reproduces_it(ctx, golden_dir, tmp_path, monkeypatch):
    z = golden(golden_dir, "main")
    agp, pairs = case_files(z, str(tmp_path))
    monkeypatch.chdir(tmp_path)
    ref_items = ast.literal_eval(str(z["pkl_args"]))
    argv = ["--bin_size", "100", "--min_len", "1"]
    for norm in ("KR", "log10", "none"):
        cap = Lines()
        plot.logger.addHandler(cap)
        try:
            plot.run(plot.parse_arguments([agp, pairs] + argv + ["--normalization", norm]), "HapHiC_plot.log", ctx=ctx)
        finally:
            plot.logger.removeHandler(cap)
        got = vmax_lines(cap.lines)
        want = list(z["log_" + norm])
        if norm == "KR":
            with open("contact_matrix.pkl", "rb") as f:
                mat, args, md5 = pickle.load(f)
            assert np.array_equal(mat, z["matrix"]) and md5 == str(z["pkl_md5"])
            assert [k for k, _ in vars(args).items()] == [k for k, _ in ref_items]
            assert [v for k, v in vars(args).items() if k not in ("agp", "alignments")] == \
                [v for k, v in ref_items if k not in ("agp", "alignments")]
        assert got[0] == want[0]
        if norm == "none":
            assert got == want
        else:
            head, tail = want[1].split(" is calculated to be ")
            gv = float(got[1].split(" is calculated to be ")[1].split(" ")[0])
            assert got[1].startswith(head) and abs(gv - float(tail.split(" ")[0])) <= 1e-9 * abs(gv)
        # the pickle as input: the same vmax lines
        cap = Lines()
        plot.logger.addHandler(cap)
        try:
            shutil.copy("contact_matrix.pkl", "in.pkl")
            plot.run(plot.parse_arguments([agp, "in.pkl"] + argv + ["--normalization", norm]), ctx=ctx)
        finally:
            plot.logger.removeHandler(cap)
        assert vmax_lines(cap.lines) == got
    assert os.path.exists("HapHiC_plot.log")


def test_kr_at_20k_bins_meets_its_stopping_rule(ctx):
    nb = 20_000
    rng = np.random.default_rng(5)
    counts = np.zeros((nb, nb), np.int64)
    idx = np.arange(nb)
    for k in range(3000):          # a distance-decay band, filled one diagonal at a time
        vals = rng.poisson(400.0 / (1.0 + k) ** 1.1, nb - k)
        counts[idx[:nb - k], idx[k:]] = vals
        counts[idx[k:], idx[:nb - k]] = vals
    (x, outer, inner, ok), = plot.kr_balance(counts, ctx=ctx)
    assert ok
    A = counts + 0.00001
    r = x * (A @ x)
    assert np.sum((1 - r) ** 2) <= 1e-12
    xo, _o, _i = plot_oracle.bnewt(A)
    np.testing.assert_allclose(x, xo, rtol=1e-6, atol=0)


def test_figures_are_written(ctx, golden_dir, tmp_path, monkeypatch):
    pytest.importorskip("matplotlib")
    z = golden(golden_dir, "main")
    agp, pairs = case_files(z, str(tmp_path))
    monkeypatch.chdir(tmp_path)
    plot.run(plot.parse_arguments([agp, pairs, "--bin_size", "100", "--separate_plots", "--output_format", "png",
                                   "--prefix", "x_"]), ctx=ctx)
    assert os.path.exists("x_contact_map.png") and os.path.exists("x_separate_plots.png")
