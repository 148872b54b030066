"""GPU parity of the two partition record formats of the link counting (hh_links.cu, "partition records"): the narrow
8-byte record {key (i << kbits) | j, flags << 29 | stream index} while the key space has at most 65,536 objects and the
stream indices stay below 2^29, the wide 16-byte one otherwise.  Every case is compared bit-exactly with the direct engine
(HH_LINKS_PARTITION=0) and with the C restatement of the counting loop, and asserts through LinkTable.record_bytes()
which format each partition set and the bucket buffer took:

  * the key-space boundary (65,536 and 65,537 contigs);
  * the stream-index boundary: a stream ending at index 2^29 - 1 and one ending at 2^29;
  * a later call whose indices cross 2^29: a narrow and a wide partition set in one finish, with a wide bucket buffer;
  * the spill list (always wide) filled from a narrow region;
  * a hot bucket and a distinct-heavy stream reaching the fallback from a narrow and from a wide bucket buffer;
  * host-staged add calls."""

import numpy as np
import pytest

from tests.test_gpu_links_buckets import (bucket_log, bucket_of, bucket_plan, forced, hot_threshold, table_slots)
from tests.test_gpu_links_partitioned import (background, count, ctx, hot_records, oracle_check, partition_of,  # noqa: F401
                                              pick_pairs, plan, planted_stream, region_cap, w)

pytestmark = pytest.mark.gpu

NARROW_END = 1 << 29            # narrow records carry stream indices below this


def check_both(ctx, w, rec, monkeypatch, lg, calls=None, offset=0, host=None):
    """Count `rec` partitioned (2^lg partitions) and directly; every output of the two and the oracle agree.  Returns
    the partitioned table."""
    forced(monkeypatch, lg)
    tab = count(ctx, w, rec, calls, offset, host)
    oracle_check(tab, w, rec, offset=offset)
    got, ctg = tab.fetch(), tab.fetch_ctg()
    monkeypatch.setenv("HH_LINKS_PARTITION", "0")
    ref = count(ctx, w, rec, calls, offset, host)
    ref.finish()
    want = ref.fetch()
    assert ref.record_bytes() == {"sets": [], "buckets": 0}
    assert sorted(got) == sorted(want)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(ctg, ref.fetch_ctg())
    ref.close()
    return tab


def fresh_flank_record(w, rec):
    """A record of a contig pair that `rec` never links, both ends at position 0 (a flank link)."""
    nx = np.nonzero(w["in_nx"] > 0)[0]
    seen = set((np.minimum(rec[:, 0], rec[:, 2]).astype(np.int64) * w["n"] + np.maximum(rec[:, 0], rec[:, 2])).tolist())
    for a in nx:
        for b in nx[::-1]:
            if a != b and int(min(a, b)) * w["n"] + int(max(a, b)) not in seen:
                return np.array([[a, 0, b, 0]], np.int32)
    raise AssertionError("no unlinked pair")


@pytest.mark.parametrize("n_ctg,nbytes", [(65_536, 8), (65_537, 16)])
def test_key_space_boundary(ctx, monkeypatch, n_ctg, nbytes):
    """The narrow key holds 2 x 16 bits: 65,536 contigs take it, 65,537 do not.  Records over 600k random pairs whose ends
    cover the whole id range, and the pairs of the highest ids."""
    from haphic_b200 import synth
    from haphic_b200.links import name_rank
    asm = synth.make_assembly(1, n_ctg, 20000, seed=81)
    assert asm.n == n_ctg
    rng = np.random.default_rng(82)
    in_nx = (rng.random(asm.n) < 0.9).astype(np.uint8)
    in_nx[-3:] = 1
    a = rng.integers(0, asm.n, 600_000)
    b = (a + rng.integers(1, asm.n, len(a))) % asm.n
    top = np.array([[n_ctg - 1, n_ctg - 2], [n_ctg - 2, n_ctg - 1], [n_ctg - 1, 0], [0, n_ctg - 1], [n_ctg - 3, n_ctg - 1]])
    a, b = np.concatenate([a, top[:, 0]]), np.concatenate([b, top[:, 1]])
    k = np.concatenate([rng.integers(0, len(a), 3_000_000), np.repeat(np.arange(len(a) - len(top), len(a)), 3)])
    L = asm.lengths
    rec = np.stack([a[k], rng.integers(0, L[a[k]]), b[k], rng.integers(0, L[b[k]])], 1).astype(np.int32)
    wd = dict(n=asm.n, lengths=L, rank=name_rank(asm.names), in_nx=in_nx)
    tab = check_both(ctx, wd, rec, monkeypatch, 5)
    assert tab.record_bytes() == {"sets": [nbytes], "buckets": nbytes}
    agg = tab.agg_info()
    assert agg["fallback_buckets"] == 0 and agg["smem_buckets"] == agg["buckets"]
    tab.close()


@pytest.mark.parametrize("end,nbytes", [(NARROW_END, 8), (NARROW_END + 1, 16)])
def test_stream_end_boundary(ctx, w, monkeypatch, end, nbytes):
    """A stream whose last index is 2^29 - 1 stays narrow, one more index makes it wide.  The last record is the first of
    its pair, so the largest first-seen index reaches the dict."""
    T = 3_000_000
    bg = background(w, T - 1)
    rec = np.concatenate([bg, fresh_flank_record(w, bg)])
    tab = check_both(ctx, w, rec, monkeypatch, 5, offset=end - T)
    assert tab.record_bytes() == {"sets": [nbytes], "buckets": nbytes}
    got = tab.fetch()
    assert int(got["first_full"].max()) == end - 1 == int(got["first_flank"][got["flank"] > 0].max())
    tab.close()


@pytest.mark.parametrize("cross", [False, True])
def test_later_call_across_narrow_end(ctx, w, monkeypatch, cross):
    """A second, small call (within the first set's slack) stays in the narrow set while its indices stay below 2^29; when
    they cross 2^29 it opens a wide set, and the finish takes both sets into a wide bucket buffer.  A planted pair
    overflows its narrow region, so the (wide) spill list holds narrow-region records too."""
    lg, T, S = 5, 4_000_000, 100_000
    pcap = region_cap(T - S, 1 << lg)
    pairs, parts = pick_pairs(w, lg, 1, seed=83)
    hot = hot_records(w, pairs, [2 * pcap], seed=84, grouped=False)
    rec = planted_stream(background(w, T - len(hot)), hot, seed=85)
    calls = [(0, T - S), (T - S, T)]
    pl = plan(w, rec[:T - S], [(0, T - S)], lg)
    assert pl["sets"][0]["fill"][parts[0]] > pcap and 0 < pl["spill"] <= pl["spill_cap"]
    offset = NARROW_END - (T - S) - (S // 2 if cross else S)
    tab = check_both(ctx, w, rec, monkeypatch, lg, calls=calls, offset=offset)
    assert tab.record_bytes() == ({"sets": [8, 16], "buckets": 16} if cross else {"sets": [8], "buckets": 8})
    tab.close()


def hot_bucket_stream(w, lg, T):
    """One contig pair with more records than the hot threshold of its bucket."""
    n_used = int((partition_of(w["pool"][:T], w["rank"], w["n"], lg) >= 0).sum())
    blog = bucket_log(n_used, lg)
    thr = hot_threshold(n_used, blog)
    pairs, _ = pick_pairs(w, blog, 1, seed=86)
    target = int(bucket_of(np.array([[pairs[0][0], 0, pairs[0][1], 0]], np.int32), w, blog)[0])
    hot = hot_records(w, pairs, [thr + 5000], seed=87, grouped=False)
    return planted_stream(background(w, T - len(hot), [target], blog), hot, seed=88), 1


def distinct_heavy_stream(w, lg, T):
    """4M records over 3.6M distinct contig pairs: most buckets hold too many distinct pairs for shared memory."""
    rng = np.random.default_rng(89)
    D = T * 9 // 10
    ii, jj = np.triu_indices(w["n"], 1)
    pick = rng.choice(len(ii), D, replace=False)
    pick = np.concatenate([pick, rng.choice(pick, T - D)])[rng.permutation(T)]
    a, b = ii[pick], jj[pick]
    flip = rng.random(T) < 0.5
    a, b = np.where(flip, b, a), np.where(flip, a, b)
    L = w["lengths"]
    rec = np.stack([a, rng.integers(0, L[a]), b, rng.integers(0, L[b])], 1).astype(np.int32)
    _, _, n_rec, n_dist = bucket_plan(w, rec, lg)
    slots = np.array([table_slots(int(n)) for n in n_rec])
    return rec, int((n_dist > slots // 4 * 3).sum())


@pytest.mark.parametrize("offset,nbytes", [(0, 8), (NARROW_END, 16)])
@pytest.mark.parametrize("stream", [hot_bucket_stream, distinct_heavy_stream], ids=["hot", "distinct"])
def test_fallback_from_either_bucket_buffer(ctx, w, monkeypatch, stream, offset, nbytes):
    """The fallback gathers its buckets' records from a narrow or a wide bucket buffer into wide records."""
    lg, T = 5, 4_000_000
    rec, n_fallback = stream(w, lg, T)
    assert n_fallback >= 1
    tab = check_both(ctx, w, rec, monkeypatch, lg, offset=offset)
    assert tab.record_bytes() == {"sets": [nbytes], "buckets": nbytes}
    agg = tab.agg_info()
    assert agg["fallback_buckets"] == n_fallback and agg["smem_buckets"] == agg["buckets"] - n_fallback
    tab.close()


@pytest.mark.parametrize("host,cross", [("numpy", False), ("pinned", True)])
def test_host_staged(ctx, w, monkeypatch, host, cross):
    """Host records staged through the two device buffers (8 Mi records each) in two calls: narrow, or with the second
    call across 2^29."""
    T, S = 10_000_000, 1_000_000
    rec = background(w, T)
    offset = NARROW_END - (T - S) - (S // 2 if cross else S)
    tab = check_both(ctx, w, rec, monkeypatch, 5, calls=[(0, T - S), (T - S, T)], offset=offset, host=host)
    assert tab.record_bytes() == ({"sets": [8, 16], "buckets": 16} if cross else {"sets": [8], "buckets": 8})
    tab.close()
