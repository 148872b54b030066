"""GPU parity of the staged scatters of the partitioned link counting (hh_k_part_scatter, hh_k_part_scatter2) at the
extremes of their runs, every field bit-exact against the C restatement of the counting loop (oracle.count_links_c).

Both kernels stage a 4096-record tile in shared memory ordered by destination and store it run by run.  The case here
has 2 partitions and 2^12 sub-buckets per region (the size of scatter2's shared histograms).  One partition region holds
nothing but a planted contig pair, so every full tile of that region is a single run of 4096 records into one sub-bucket.
The other region receives all the background records and overflows, so the scatter tile that crosses the region's
capacity has a run that is cut in the middle: its head goes to the region, its tail to the spill list."""

import numpy as np
import pytest

from tests.test_gpu_links_buckets import bucket_of, bucket_plan, forced
from tests.test_gpu_links_partitioned import (FLANK_BP, count, ctx, hot_records, oracle_check,  # noqa: F401
                                              partition_of, pick_pairs, plan, planted_stream, report, w)

pytestmark = pytest.mark.gpu

TILE = 4096


def test_one_sub_bucket_tiles_with_4096_sub_buckets(ctx, w, monkeypatch):
    from haphic_b200 import synth
    lg, T, H = 1, 10_000_000, 5 * TILE + 123
    forced(monkeypatch, lg)
    pairs, parts = pick_pairs(w, lg, 1, seed=51)
    hot = hot_records(w, pairs, [H], seed=52, grouped=True)
    # usable background records of the other partition only (about 28 % of the generator's records)
    pool = synth.make_pairs(w["asm"], 40_000_000, seed=54, device="cuda").cpu().numpy()
    bg = pool[partition_of(pool, w["rank"], w["n"], lg) == 1 - parts[0]][:T - H]
    del pool
    assert len(bg) == T - H
    rec = planted_stream(bg, hot, seed=53, run_at=(T - H) // 3)
    pl = plan(w, rec, [(0, T)], lg)
    report("one sub-bucket tiles", pl)
    fill = pl["sets"][0]["fill"]
    assert fill[parts[0]] == H                              # the planted region holds the planted pair alone
    assert 0 < pl["spill"] <= pl["spill_cap"]               # the other region overflows into the spill list
    blog, thr, n_rec, n_dist = bucket_plan(w, rec, lg)
    target = int(bucket_of(hot[:1], w, blog)[0])
    print("{} buckets, {} per region; planted bucket {}: {} records, {} pairs".format(
        1 << blog, 1 << (blog - lg), target, n_rec[target], n_dist[target]))
    assert blog - lg == 12 and n_rec[target] == H and n_rec[target] <= thr
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    agg = tab.agg_info()
    assert agg["buckets"] == 1 << blog
    tab.close()
