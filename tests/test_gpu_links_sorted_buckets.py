"""GPU parity of the sort-and-reduce bucket count of the partitioned link counting (hh_links.cu, hh_k_bucket_count) at
the edges of its chunks, every field bit-exact against the C restatement of the counting loop (oracle.count_links_c):

  * a bucket of exactly one chunk of records (2048 with 32-bit keys), and one of a chunk + 1, where the record of the
    second chunk belongs to a pair that also has records in the first, so the second chunk merges into the list;
  * a bucket of several chunks with one heavy pair and exactly the distinct-pair limit, counted in shared memory, and the
    same with one pair more, which falls back;
  * more than 65,535 contigs, where the sort key (i << kbits) | j is wider than 32 bits.

Every case asserts through LinkTable.agg_info() that the path it targets ran."""

import numpy as np
import pytest

from tests.test_gpu_links_buckets import AGG_LIMIT, bucket_log, bucket_plan, distinct_pairs_in_bucket, forced
from tests.test_gpu_links_partitioned import FLANK_BP, background, count, ctx, oracle_check, partition_of, planted_stream, w  # noqa: F401

pytestmark = pytest.mark.gpu

CHUNK32 = 2048                          # records per chunk with 32-bit keys (256 threads x 8)
CHUNK64 = 1280                          # with 64-bit keys (256 threads x 5)


def pair_records(w, a, b, cnt, seed):
    """cnt records of the pair (a, b): each end at the start, a quarter, the middle or the end of its contig (flank and
    non-flank, head and tail), half of them with the ends swapped."""
    rng = np.random.default_rng(seed)
    L = w["lengths"]
    flip = rng.random(cnt) < 0.5
    r = np.empty((cnt, 4), np.int32)
    r[:, 0], r[:, 2] = np.where(flip, b, a), np.where(flip, a, b)
    for col, ctg in ((1, r[:, 0]), (3, r[:, 2])):
        ln = L[ctg]
        choices = np.stack([np.zeros_like(ln), ln // 4, ln // 2, ln - 1], 1)
        r[:, col] = choices[np.arange(cnt), rng.integers(0, 4, cnt)]
    return r


def one_bucket_stream(w, lg, T, n_pairs, counts, seed):
    """A background of about T records that avoids one bucket, and that bucket planted with n_pairs distinct pairs, pair k
    with counts[k] records.  Returns the stream, the bucket and the bucket plan."""
    n_used = int((partition_of(w["pool"][:T], w["rank"], w["n"], lg) >= 0).sum())
    blog = bucket_log(n_used, lg)
    a, b, target = distinct_pairs_in_bucket(w, blog, n_pairs, seed=seed)
    hot = np.concatenate([pair_records(w, a[k], b[k], int(counts[k]), seed + 1 + k) for k in range(n_pairs)])
    rec = planted_stream(background(w, T - len(hot), [target], blog), hot, seed=seed)
    blog2, thr, n_rec, n_dist = bucket_plan(w, rec, lg)
    assert blog2 == blog and n_rec[target] == len(hot) and n_dist[target] == n_pairs and n_rec[target] < thr
    return rec, target, n_rec, n_dist


@pytest.mark.parametrize("extra", [0, 1])
def test_bucket_of_one_chunk_and_one_more_record(ctx, w, monkeypatch, extra):
    """A bucket of CHUNK32 + extra records: two heavy pairs and 300 pairs of two records each.  Every pair has at least two
    records, so with extra = 1 the one record of the second chunk always belongs to a pair of the first."""
    lg, T = 5, 4_000_000
    forced(monkeypatch, lg)
    small = 300
    heavy = CHUNK32 + extra - 2 * small
    counts = [heavy - heavy // 2, heavy // 2] + [2] * small
    rec, target, n_rec, n_dist = one_bucket_stream(w, lg, T, small + 2, counts, seed=51)
    print("\nbucket {}: {} records / {} pairs".format(target, n_rec[target], n_dist[target]))
    assert n_rec[target] == CHUNK32 + extra
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    agg = tab.agg_info()
    assert agg["fallback_buckets"] == 0 and agg["smem_buckets"] == agg["buckets"]
    tab.close()


@pytest.mark.parametrize("extra", [0, 1])
def test_many_chunks_at_the_distinct_pair_limit(ctx, w, monkeypatch, extra):
    """A bucket of several chunks: one pair with 6000 records and AGG_LIMIT - 1 + extra pairs of two records each,
    interleaved, so later chunks both add to pairs already on the list and bring new ones.  At the limit it is counted in
    shared memory; one pair more and it falls back."""
    lg, T = 5, 4_000_000
    forced(monkeypatch, lg)
    n_pairs = AGG_LIMIT + extra
    rec, target, n_rec, n_dist = one_bucket_stream(w, lg, T, n_pairs, [6000] + [2] * (n_pairs - 1), seed=61)
    print("\nlimit +{}: bucket {} holds {} records ({} chunks) / {} pairs".format(
        extra, target, n_rec[target], -(-n_rec[target] // CHUNK32), n_dist[target]))
    assert n_rec[target] > 3 * CHUNK32
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    agg = tab.agg_info()
    assert agg["fallback_buckets"] == extra and agg["smem_buckets"] == agg["buckets"] - extra
    tab.close()


def test_more_than_65535_contigs(ctx, monkeypatch):
    """70,000 contigs: the key needs 2 x 17 bits.  Records are drawn from 1M random pairs (about four per pair, so the
    buckets are counted in shared memory, most of them in two chunks) whose ends cover the whole id range."""
    from haphic_b200 import synth
    from haphic_b200.links import name_rank
    forced(monkeypatch, 5)
    asm = synth.make_assembly(8, 70_000, 20000, seed=71)
    rng = np.random.default_rng(72)
    in_nx = (rng.random(asm.n) < 0.9).astype(np.uint8)
    a = rng.integers(0, asm.n, 1_000_000)
    b = (a + rng.integers(1, asm.n, len(a))) % asm.n
    k = rng.integers(0, len(a), 4_000_000)
    L = asm.lengths
    rec = np.stack([a[k], rng.integers(0, L[a[k]]), b[k], rng.integers(0, L[b[k]])], 1).astype(np.int32)
    wide = dict(n=asm.n, lengths=L, rank=name_rank(asm.names), in_nx=in_nx)
    _, _, n_rec, n_dist = bucket_plan(wide, rec, 5)
    assert (n_dist <= AGG_LIMIT).all() and n_rec.max() > CHUNK64
    assert rec[:, [0, 2]].max() >= 1 << 16
    tab = count(ctx, wide, rec)
    oracle_check(tab, wide, rec)
    agg = tab.agg_info()
    assert agg["fallback_buckets"] == 0 and agg["smem_buckets"] == agg["buckets"]
    tab.close()
