"""GPU parity of the bucket aggregation of the partitioned link counting (hh_links.cu, hh_k_bucket_count and its
fallback), every field bit-exact against the C restatement of the counting loop (oracle.count_links_c):

  * a bucket planted with one distinct contig pair more than its shared-memory table takes (it is abandoned and recounted
    by the global-table fallback), and one planted exactly at that limit (counted in shared memory).  The planted pairs
    carry flank links, so an abandoned bucket that left a trace would count per-contig totals or nnz_flank twice;
  * a bucket above the record threshold made of one hot contig pair (it bypasses shared memory);
  * a stream of nearly all-distinct contig pairs, where most buckets are abandoned and the fallback counts them in
    several batches;
  * 2 and 1024 partitions (the fan-out of a partition into buckets at its extremes);
  * streams shaped like the benchmark's (50k contigs, its generator), at 32M records against the oracle and at the
    benchmark's 200M records against the direct engine, where no bucket may fall back.

Planted pairs are placed in chosen buckets with a numpy port of the bucket rule (the top bucket_log bits of hh_mix64 of
the key, links_bucket_log), and every case asserts through LinkTable.agg_info() that the path it targets ran."""

import numpy as np
import pytest
import torch

from tests.test_gpu_links_partitioned import (FLANK_BP, assert_equals_oracle, background, count, ctx, hot_records,  # noqa: F401
                                              oracle_check, partition_of, pick_pairs, planted_stream, w)

pytestmark = pytest.mark.gpu

AGG_MEAN, SUB_MAX_LOG, AGG_SLOTS, AGG_HOT, AGG_THREADS = 2048, 12, 2048, 32, 256
FB_BATCH = 1 << 19                      # records per fallback batch (HH_FB_BATCH)
AGG_LIMIT = AGG_SLOTS // 4 * 3          # distinct pairs a full-size shared-memory table takes


# ---- the bucket rules of hh_links.cu, restated ------------------------------------------------------------------------

def bucket_log(n_used, npart_log):
    """links_bucket_log: a mean of at most 2048 records per bucket, 1 .. 2^12 buckets per partition."""
    b = npart_log
    while b < npart_log + SUB_MAX_LOG and (n_used >> b) > AGG_MEAN:
        b += 1
    return b


def hot_threshold(n_used, blog):
    """links_hot_records: 32 x the mean bucket, at least 32 x 1024 records."""
    mean = (n_used + (1 << blog) - 1) >> blog
    return AGG_HOT * max(mean, AGG_MEAN // 2)


def table_slots(n_rec):
    """Slots of a bucket's shared-memory table (hh_k_bucket_count): the power of two >= 1.5 x its records, 256 .. 2048."""
    t = AGG_THREADS
    while t < AGG_SLOTS and t * 2 < n_rec * 3:
        t <<= 1
    return t


def bucket_of(rec, w, blog):
    """Bucket of every record (the top blog bits of the key hash); -1 = not a usable record."""
    return partition_of(rec, w["rank"], w["n"], blog)


def ordered_key(rec, w):
    a, b = rec[:, 0].astype(np.int64), rec[:, 2].astype(np.int64)
    swap = w["rank"][a] > w["rank"][b]
    return np.where(swap, b, a) * w["n"] + np.where(swap, a, b)


def bucket_plan(w, rec, lg):
    """(bucket_log, hot threshold, records per bucket, distinct pairs per bucket) of a stream."""
    blog = bucket_log(int((bucket_of(rec, w, 1) >= 0).sum()), lg)
    bk = bucket_of(rec, w, blog)
    used = bk >= 0
    nb = 1 << blog
    n_rec = np.bincount(bk[used], minlength=nb)
    key = ordered_key(rec[used], w)
    _, first = np.unique(key, return_index=True)
    n_dist = np.bincount(bk[used][first], minlength=nb)
    return blog, hot_threshold(int(used.sum()), blog), n_rec, n_dist


def forced(monkeypatch, lg):
    monkeypatch.setenv("HH_LINKS_PARTITION", "1")
    monkeypatch.setenv("HH_LINKS_NPART_LOG", str(lg))


def distinct_pairs_in_bucket(w, blog, k, seed):
    """k distinct Nx contig pairs of one bucket, and that bucket."""
    nx = np.nonzero(w["in_nx"] > 0)[0]
    ii, jj = np.triu_indices(len(nx), 1)
    cand = np.stack([nx[ii], np.zeros_like(ii), nx[jj], np.zeros_like(ii)], 1).astype(np.int32)
    bk = bucket_of(cand, w, blog)
    target = int(np.argmax(np.bincount(bk)))
    sel = np.nonzero(bk == target)[0]
    assert len(sel) >= k, (len(sel), k)
    sel = np.random.default_rng(seed).choice(sel, k, replace=False)
    return cand[sel, 0], cand[sel, 2], target


def flank_records(w, a, b):
    """Two records per pair: both ends at position 0 (a flank link whenever both contigs are in Nx), then both ends
    mid-contig; the first one comes first in the stream, so first_flank = first_full."""
    L = w["lengths"]
    r1 = np.stack([a, np.zeros_like(a), b, np.zeros_like(b)], 1)
    r2 = np.stack([b, L[b] // 2, a, L[a] // 2], 1)
    return np.concatenate([r1, r2]).astype(np.int32)


# ---- the shared-memory table's limit and the fallback -----------------------------------------------------------------

@pytest.mark.parametrize("extra", [0, 1])
def test_distinct_pair_limit(ctx, w, monkeypatch, extra):
    """One bucket with exactly AGG_LIMIT distinct flank-linked pairs is counted in shared memory; one more pair and it is
    abandoned and recounted by the fallback, with per-contig totals and nnz_flank counted once."""
    lg, T = 5, 4_000_000
    forced(monkeypatch, lg)
    n_used = int((partition_of(w["pool"][:T], w["rank"], w["n"], lg) >= 0).sum())
    blog = bucket_log(n_used, lg)
    a, b, target = distinct_pairs_in_bucket(w, blog, AGG_LIMIT + extra, seed=31)
    hot = flank_records(w, a, b)
    rec = planted_stream(background(w, T - len(hot), [target], blog), hot, seed=33)
    blog2, thr, n_rec, n_dist = bucket_plan(w, rec, lg)
    print("\nlimit +{}: {} buckets, bucket {} holds {} records / {} pairs, others at most {} pairs".format(
        extra, 1 << blog2, target, n_rec[target], n_dist[target], np.delete(n_dist, target).max()))
    assert blog2 == blog and n_dist[target] == AGG_LIMIT + extra and n_rec[target] < thr
    assert np.delete(n_dist, target).max() <= AGG_LIMIT and n_rec.max() <= thr
    tab = count(ctx, w, rec)
    ref = oracle_check(tab, w, rec)
    assert len(ref["flank_vals"]) >= AGG_LIMIT
    agg = tab.agg_info()
    assert agg["buckets"] == 1 << blog
    assert agg["fallback_buckets"] == extra and agg["smem_buckets"] == agg["buckets"] - extra
    tab.close()


def test_hot_bucket_bypasses_shared_memory(ctx, w, monkeypatch):
    """One contig pair with more records than the threshold: its bucket goes straight to the fallback."""
    lg, T = 5, 4_000_000
    forced(monkeypatch, lg)
    n_used = int((partition_of(w["pool"][:T], w["rank"], w["n"], lg) >= 0).sum())
    blog = bucket_log(n_used, lg)
    thr = hot_threshold(n_used, blog)
    pairs, _ = pick_pairs(w, blog, 1, seed=34)
    target = int(bucket_of(np.array([[pairs[0][0], 0, pairs[0][1], 0]], np.int32), w, blog)[0])
    hot = hot_records(w, pairs, [thr + 5000], seed=35, grouped=False)
    rec = planted_stream(background(w, T - len(hot), [target], blog), hot, seed=36)
    blog2, thr2, n_rec, n_dist = bucket_plan(w, rec, lg)
    print("\nhot bucket: {} records over a threshold of {}".format(n_rec[target], thr2))
    assert blog2 == blog and n_rec[target] > thr2 and n_dist[target] == 1
    assert np.delete(n_rec, target).max() <= thr2 and n_dist.max() <= AGG_LIMIT
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    agg = tab.agg_info()
    assert agg["fallback_buckets"] == 1 and agg["smem_buckets"] == agg["buckets"] - 1
    tab.close()


def test_distinct_heavy_stream_falls_back_in_batches(ctx, w, monkeypatch):
    """4M records over 3.6M distinct contig pairs (of the 4.5M there are): nearly every bucket holds more distinct pairs
    than 3/4 of its table, is abandoned and counted by the fallback, whose gathered records span several batches."""
    lg, T, D = 5, 4_000_000, 3_600_000
    forced(monkeypatch, lg)
    rng = np.random.default_rng(37)
    ii, jj = np.triu_indices(w["n"], 1)
    pick = rng.choice(len(ii), D, replace=False)
    pick = np.concatenate([pick, rng.choice(pick, T - D)])[rng.permutation(T)]
    a, b = ii[pick], jj[pick]
    flip = rng.random(T) < 0.5
    a, b = np.where(flip, b, a), np.where(flip, a, b)
    L = w["lengths"]
    rec = np.stack([a, rng.integers(0, L[a]), b, rng.integers(0, L[b])], 1).astype(np.int32)
    blog, thr, n_rec, n_dist = bucket_plan(w, rec, lg)
    slots = np.array([table_slots(int(n)) for n in n_rec])
    abandoned = n_dist > slots // 4 * 3
    fb_records = int(n_rec[abandoned].sum())
    print("\ndistinct-heavy: {} of {} buckets abandoned, {} records in the fallback ({} batches of at most {})".format(
        int(abandoned.sum()), 1 << blog, fb_records, -(-fb_records // FB_BATCH), FB_BATCH))
    assert n_rec.max() <= thr and abandoned.sum() > (1 << blog) * 3 // 4 and fb_records > 4 * FB_BATCH
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    agg = tab.agg_info()
    assert agg["buckets"] == 1 << blog
    assert agg["fallback_buckets"] == int(abandoned.sum()) and agg["smem_buckets"] == agg["buckets"] - agg["fallback_buckets"]
    tab.close()


@pytest.mark.parametrize("lg", [1, 10])
def test_fan_out_extremes(ctx, w, monkeypatch, lg):
    """2 partitions (1024 buckets each) and 1024 partitions (2 buckets each): every bucket in shared memory."""
    T = 4_000_000
    forced(monkeypatch, lg)
    rec = np.ascontiguousarray(w["pool"][:T])
    blog, thr, n_rec, n_dist = bucket_plan(w, rec, lg)
    print("\n{} partitions: {} buckets, {} per partition".format(1 << lg, 1 << blog, 1 << (blog - lg)))
    assert blog - lg == (10 if lg == 1 else 1)
    assert n_rec.max() <= thr and n_dist.max() <= AGG_LIMIT
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    assert tab.agg_info() == {"buckets": 1 << blog, "smem_buckets": 1 << blog, "fallback_buckets": 0}
    tab.close()


def test_direct_table_reports_no_buckets(ctx, w, monkeypatch):
    monkeypatch.setenv("HH_LINKS_PARTITION", "0")
    rec = np.ascontiguousarray(w["pool"][:100_000])
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    assert tab.agg_info() == {"buckets": 0, "smem_buckets": 0, "fallback_buckets": 0}
    tab.close()


# ---- the benchmark's shape ----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def c3():
    from haphic_b200 import synth
    from haphic_b200.links import name_rank
    asm = synth.make_assembly(24, 50000, 20000, seed=12345)
    return dict(asm=asm, rank=name_rank(asm.names), in_nx=np.ones(asm.n, np.uint8))


def c3_table(ctx, c3, rec):
    from haphic_b200.links import LinkTable
    P = int(rec.shape[0])
    tab = LinkTable(ctx, c3["asm"].lengths, c3["rank"], c3["in_nx"], 500000, capacity_hint=int(0.45 * P))
    tab.add(rec, asynchronous=True)
    return tab, tab.finish()


def test_c3_shape_against_oracle(ctx, c3, monkeypatch):
    """32M records of the benchmark's generator on its 50k contigs, the default engine choice (partitioned)."""
    from haphic_b200 import synth
    monkeypatch.delenv("HH_LINKS_PARTITION", raising=False)
    monkeypatch.delenv("HH_LINKS_NPART_LOG", raising=False)
    rec = synth.make_pairs_range(c3["asm"], 0, 32_000_000, seed=12346, device="cuda")
    tab, info = c3_table(ctx, c3, rec)
    agg = tab.agg_info()
    print("\n32M records: {} used, {} buckets, {} fallback".format(info.n_used, agg["buckets"], agg["fallback_buckets"]))
    assert agg["buckets"] == 1 << bucket_log(int(info.n_used), 7)
    assert agg["fallback_buckets"] == 0 and agg["smem_buckets"] == agg["buckets"]
    assert_equals_oracle(tab, info, rec.cpu().numpy(), c3["asm"].lengths, c3["rank"], c3["in_nx"], 500000)
    tab.close()


def test_c3_full_size_no_fallback(ctx, c3, monkeypatch):
    """The benchmark's 200M records: 2^17 buckets, none falls back, and every field equals the direct engine's."""
    from haphic_b200 import synth
    monkeypatch.delenv("HH_LINKS_NPART_LOG", raising=False)
    monkeypatch.delenv("HH_LINKS_PARTITION", raising=False)
    rec = synth.make_pairs_range(c3["asm"], 0, 200_000_000, seed=12346, device="cuda")
    tab, info = c3_table(ctx, c3, rec)
    agg = tab.agg_info()
    print("\n200M records: {} used, {} buckets, {} fallback".format(info.n_used, agg["buckets"], agg["fallback_buckets"]))
    assert agg == {"buckets": 1 << 17, "smem_buckets": 1 << 17, "fallback_buckets": 0}
    got, tot = tab.fetch(), tab.fetch_ctg()
    tab.close()
    monkeypatch.setenv("HH_LINKS_PARTITION", "0")
    ref_tab, ref_info = c3_table(ctx, c3, rec)
    assert (info.n_used, info.nnz_full, info.nnz_flank) == (ref_info.n_used, ref_info.nnz_full, ref_info.nnz_flank)
    ref = ref_tab.fetch()
    for k in ref:
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(tot, ref_tab.fetch_ctg())
    ref_tab.close()
    del rec
    torch.cuda.empty_cache()
