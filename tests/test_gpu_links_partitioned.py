"""GPU parity of the link counting (hh_links.cu) on the paths the plain synthetic streams never reach, every field
bit-exact against the C restatement of the counting loop (oracle.count_links_c):

  * the spill list of the partitioned count: contig pairs planted so often that their partition region overflows, at the
    region boundary (pcap records fit, pcap + 1 spill one) and at the spill list's own capacity;
  * a stream sent in several calls that open several partition sets, whose spill must fit as it does in one call;
  * a truly over-capacity stream: a clear error, and the direct engine counts the same stream;
  * double-buffered host staging over several chunks and calls, from numpy and from pinned memory;
  * partition counts at the extremes (2 and 1024 partitions, and the clamping of values outside them);
  * the default engine choice at its thresholds (16 Mi records, 2048 contigs);
  * stream indices across 2^31 and up to the last index the API accepts, through the dict order, the linked index and the
    matrix.

Planted pairs are placed in chosen partitions with a numpy port of hh_mix64, and every planted case asserts the partition
fills and spill it relies on, computed from the sizing rules of hh_links.cu (links_new_partset, links_size_spill,
links_choose_mode), so a change of those rules fails here instead of silently dropping the coverage.  Run with -s to see
the predicted fills and spill of every case."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NONE32 = 0xFFFFFFFF
FLANK_BP = 5000
N_CTG, N_CHR, MEAN_LEN, POOL, SEED = 3000, 8, 30000, 24_000_000, 4242


# ---- the partition sizing of hh_links.cu, restated -------------------------------------------------------------------

def mix64(k):
    """hh_mix64 (and mix64 of oracle/haphic_oracle.c): the key hash whose high bits pick the partition."""
    k = np.asarray(k, dtype=np.uint64)
    k = k ^ (k >> np.uint64(33))
    k = k * np.uint64(0xFF51AFD7ED558CCD)
    k = k ^ (k >> np.uint64(33))
    k = k * np.uint64(0xC4CEB9FE1A85EC53)
    return k ^ (k >> np.uint64(33))


def partition_of(rec, rank, n_ctg, npart_log):
    """Partition of every record (hh_k_part_scatter: name-ordered ends, key (i << 32) | j); -1 = not a usable record."""
    a, b = rec[:, 0].astype(np.int64), rec[:, 2].astype(np.int64)
    ok = (a != b) & (a >= 0) & (a < n_ctg) & (b >= 0) & (b < n_ctg)
    a, b = np.where(ok, a, 0), np.where(ok, b, 0)
    swap = rank[a] > rank[b]
    i, j = np.where(swap, b, a), np.where(swap, a, b)
    key = (i.astype(np.uint64) << np.uint64(32)) | j.astype(np.uint64)
    p = (mix64(key) >> np.uint64(64 - npart_log)).astype(np.int64)
    return np.where(ok, p, -1)


def region_cap(n_rec, npart):
    """Records per partition region of a set sized for n_rec records (links_new_partset)."""
    return int(n_rec / npart * 1.5) + 4096


def spill_cap(sized):
    """Spill list entries for partition sets sized for `sized` records in all (links_size_spill)."""
    return int(sum(sized)) // 8 + (4 << 20)


def default_npart_log(total):
    """links_choose_mode: about 400k records per partition, 16 to 512 partitions."""
    lg = 4
    while lg < 9 and (400000 << lg) < total:
        lg += 1
    return lg


def plan(w, rec, calls, npart_log):
    """The partition sets the calls open (links_part_room), their region fills and the records that spill."""
    npart = 1 << npart_log
    part = partition_of(rec, w["rank"], w["n"], npart_log)
    sets = []
    for lo, hi in calls:
        m = hi - lo
        if not sets or sets[-1]["sent"] + m <= sets[-1]["sized"] + sets[-1]["sized"] // 8:
            if not sets:
                sets.append(dict(sized=m, sent=0, parts=[]))
            sets[-1]["sent"] += m
        else:
            sets.append(dict(sized=m, sent=m, parts=[]))
        sets[-1]["parts"].append(part[lo:hi])
    for s in sets:
        p = np.concatenate(s["parts"])
        s["fill"] = np.bincount(p[p >= 0], minlength=npart)
        s["pcap"] = region_cap(s["sized"], npart)
        s["spill"] = int(np.maximum(s["fill"] - s["pcap"], 0).sum())
        del s["parts"]
    out = dict(npart=npart, sets=sets, spill=sum(s["spill"] for s in sets), spill_cap=spill_cap([s["sized"] for s in sets]))
    return out


def report(name, pl):
    sets = ", ".join("pcap {} max fill {} spill {}".format(s["pcap"], int(s["fill"].max()), s["spill"]) for s in pl["sets"])
    print("\n{}: {} partitions; {}; predicted spill {} of spill list {}".format(name, pl["npart"], sets, pl["spill"],
                                                                             pl["spill_cap"]))


# ---- the oracle comparison --------------------------------------------------------------------------------------------

def assert_equals_oracle(tab, info, rec, lengths, rank, in_nx, flank_bp, offset=0, cap=None):
    """Every counter of a finished table against oracle.count_links_c of the same records streamed from `offset`:
    keys in dict insertion order, full / first_full, flank in flank-dict order / first_flank (NONE32 where a pair has
    no flank link), the HH / HT / TH / TT split, the per-contig totals, n_used, nnz_full and nnz_flank.  Returns the
    oracle's arrays."""
    from oracle import haphic_oracle as orc
    ref = orc.count_links_c(rec, lengths, rank, in_nx, flank_bp, cap=cap)
    assert info.n_used == ref["n_used"]
    assert info.nnz_full == len(ref["full_vals"]) and info.nnz_flank == len(ref["flank_vals"])
    got = tab.fetch()
    assert np.array_equal(np.stack([got["key_i"], got["key_j"]], 1), ref["full_keys"])
    assert np.array_equal(got["full"].astype(np.int64), ref["full_vals"])
    assert np.array_equal(got["first_full"].astype(np.int64), ref["full_first"] + offset)
    sel = np.nonzero(got["flank"] > 0)[0]
    sel = sel[np.argsort(got["first_flank"][sel], kind="stable")]
    assert np.array_equal(np.stack([got["key_i"][sel], got["key_j"][sel]], 1), ref["flank_keys"])
    assert np.array_equal(got["flank"][sel].astype(np.int64), ref["flank_vals"])
    assert np.array_equal(got["first_flank"][sel].astype(np.int64), ref["flank_first"] + offset)
    assert (got["first_flank"][got["flank"] == 0] == NONE32).all()
    assert np.array_equal(got["ht"].astype(np.int64), ref["ht"])
    assert np.array_equal(tab.fetch_ctg(), ref["ctg_link_total"])
    return ref


# ---- streams with planted pairs ---------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ctx():
    from haphic_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def w():
    """A few thousand contigs, 10 % of them outside Nx, and a pool of synthetic background records."""
    from haphic_b200 import synth
    from haphic_b200.links import name_rank
    asm = synth.make_assembly(N_CHR, N_CTG, MEAN_LEN, seed=SEED)
    rng = np.random.default_rng(SEED)
    in_nx = (rng.random(asm.n) < 0.9).astype(np.uint8)
    pool = synth.make_pairs(asm, POOL, seed=SEED + 1, device="cuda").cpu().numpy()
    # planted pairs join long Nx contigs, so that they have flank and non-flank, head and tail positions
    eligible = np.nonzero((asm.lengths >= 4 * FLANK_BP) & (in_nx > 0))[0]
    return dict(asm=asm, n=asm.n, lengths=asm.lengths, rank=name_rank(asm.names), in_nx=in_nx, pool=pool, eligible=eligible)


def pick_pairs(w, npart_log, k, seed, upper_first=False):
    """k contig pairs of k distinct partitions; with upper_first the first lies in the upper half of the partitions."""
    rng = np.random.default_rng(seed)
    npart = 1 << npart_log
    pairs, parts = [], set()
    while len(pairs) < k:
        a, b = (int(x) for x in rng.choice(w["eligible"], 2, replace=False))
        p = int(partition_of(np.array([[a, 0, b, 0]], np.int32), w["rank"], w["n"], npart_log)[0])
        if p in parts or (upper_first and not pairs and p < npart // 2):
            continue
        pairs.append((a, b))
        parts.add(p)
    return pairs, sorted(parts)


def hot_records(w, pairs, counts, seed, grouped):
    """`counts[k]` records of pair k: each end at a flank head, mid-contig head, mid-contig tail or flank tail position,
    half of them with the ends swapped.  The first record of every pair has both ends mid-contig (no flank link), so its
    first_flank differs from first_full.  grouped=True keeps each pair's records together (runs of one key)."""
    rng = np.random.default_rng(seed)
    L = w["lengths"]
    out = []
    for (a, b), cnt in zip(pairs, counts):
        ends = np.array([a, b])
        r = np.empty((cnt, 4), np.int32)
        flip = rng.random(cnt) < 0.5
        r[:, 0], r[:, 2] = np.where(flip, b, a), np.where(flip, a, b)
        for col, ctg in ((1, r[:, 0]), (3, r[:, 2])):
            ln = L[ctg]
            choices = np.stack([np.zeros_like(ln), ln // 2 - 100, ln // 2 + 100, ln - 1], 1)
            r[:, col] = choices[np.arange(cnt), rng.integers(0, 4, cnt)]
        assert set(np.unique(r[:, [0, 2]]).tolist()) == set(ends.tolist())
        out.append(r)
    hot = np.concatenate(out)
    if not grouped:
        hot = hot[rng.permutation(len(hot))]
    key = np.minimum(hot[:, 0], hot[:, 2]).astype(np.int64) * w["n"] + np.maximum(hot[:, 0], hot[:, 2])
    _, first = np.unique(key, return_index=True)
    hot[first, 1] = L[hot[first, 0]] // 2 - 100
    hot[first, 3] = L[hot[first, 2]] // 2 + 100
    return hot


def background(w, n, avoid_parts=(), npart_log=0):
    """n pool records, without those of the partitions in avoid_parts (so a planted partition holds the planted records
    only)."""
    pool = w["pool"]
    if avoid_parts:
        p = partition_of(pool, w["rank"], w["n"], npart_log)
        pool = pool[~np.isin(p, list(avoid_parts))]
    assert len(pool) >= n
    return pool[:n]


def planted_stream(bg, hot, seed, run_at=None):
    """bg with the hot records interleaved at random places, or as one contiguous run starting at run_at."""
    n = len(bg) + len(hot)
    if run_at is None:
        pos = np.sort(np.random.default_rng(seed).choice(n, len(hot), replace=False))
    else:
        pos = np.arange(run_at, run_at + len(hot))
    mask = np.zeros(n, bool)
    mask[pos] = True
    out = np.empty((n, 4), np.int32)
    out[mask] = hot
    out[~mask] = bg
    return out


def count(ctx, w, rec, calls=None, offset=0, host=None, asynchronous=False):
    """A table of `rec` streamed from `offset` in the given calls: device tensors, or host memory ("numpy" / "pinned")."""
    from haphic_b200.links import LinkTable
    tab = LinkTable(ctx, w["lengths"], w["rank"], w["in_nx"], FLANK_BP)
    for lo, hi in (calls or [(0, len(rec))]):
        part = np.ascontiguousarray(rec[lo:hi])
        if host == "numpy":
            chunk = part
        elif host == "pinned":
            chunk = torch.from_numpy(part).pin_memory()
        else:
            chunk = torch.from_numpy(part).cuda()
        tab.add(chunk, stream_offset=offset + lo, asynchronous=asynchronous)
    return tab


def oracle_check(tab, w, rec, offset=0):
    info = tab.finish()
    return assert_equals_oracle(tab, info, rec, w["lengths"], w["rank"], w["in_nx"], FLANK_BP, offset=offset)


@pytest.fixture
def partitioned(monkeypatch):
    """Forced partitioned counting with 2^lg partitions."""
    def set_lg(lg):
        monkeypatch.setenv("HH_LINKS_PARTITION", "1")
        monkeypatch.setenv("HH_LINKS_NPART_LOG", str(lg))
    return set_lg


@pytest.fixture(params=["direct", "partitioned"])
def counting_mode(request, monkeypatch):
    monkeypatch.setenv("HH_LINKS_PARTITION", "1" if request.param == "partitioned" else "0")
    monkeypatch.setenv("HH_LINKS_NPART_LOG", "5")
    return request.param


# ---- the spill list ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("layout", ["interleaved", "run"])
def test_spill_one_call(ctx, w, partitioned, layout):
    """Three planted pairs in three partitions: one overflows its region several times over, two by less.  Interleaved
    with the background, or one contiguous run (warps of 32 equal keys in the spill scan)."""
    lg, T = 5, 16_000_000
    partitioned(lg)
    pcap = region_cap(T, 1 << lg)
    pairs, parts = pick_pairs(w, lg, 3, seed=1)
    counts = [4 * pcap, 3 * pcap // 2, pcap + 1000]
    hot = hot_records(w, pairs, counts, seed=2, grouped=layout == "run")
    rec = planted_stream(background(w, T - len(hot)), hot, seed=3, run_at=None if layout == "interleaved" else T // 3)
    pl = plan(w, rec, [(0, T)], lg)
    report("spill, one call, " + layout, pl)
    fill = pl["sets"][0]["fill"]
    assert pl["sets"][0]["pcap"] == pcap and fill.max() > 3 * pcap
    assert (fill[parts] > pcap).all() and (np.delete(fill, parts) <= pcap).all()
    assert pl["spill"] <= pl["spill_cap"]
    ref = oracle_check(count(ctx, w, rec), w, rec)
    # the planted pairs are first seen without a flank link: first_flank and first_full differ
    full_first = dict(zip(map(tuple, ref["full_keys"].tolist()), ref["full_first"].tolist()))
    flank_first = dict(zip(map(tuple, ref["flank_keys"].tolist()), ref["flank_first"].tolist()))
    for a, b in pairs:
        k = (a, b) if w["rank"][a] < w["rank"][b] else (b, a)
        assert flank_first[k] > full_first[k]


def test_spill_region_boundary(ctx, w, partitioned):
    """One partition filled to exactly pcap records (no spill) and one to pcap + 1 (one record spills): q < pcap."""
    lg, T = 5, 4_000_000
    partitioned(lg)
    pcap = region_cap(T, 1 << lg)
    pairs, parts = pick_pairs(w, lg, 2, seed=4)
    hot = hot_records(w, pairs, [pcap, pcap + 1], seed=5, grouped=False)
    rec = planted_stream(background(w, T - len(hot), parts, lg), hot, seed=6)
    pl = plan(w, rec, [(0, T)], lg)
    report("region boundary", pl)
    fill = pl["sets"][0]["fill"]
    assert sorted(fill[parts].tolist()) == [pcap, pcap + 1] and pl["spill"] == 1
    assert np.delete(fill, parts).max() < pcap
    oracle_check(count(ctx, w, rec), w, rec)


@pytest.mark.parametrize("over", [0, 1])
def test_spill_list_boundary(ctx, w, partitioned, over):
    """The spill list filled to exactly its capacity counts exactly; one record more is refused with HH_ERR_CAPACITY.
    Together the two pin the number of records that actually spill to the predicted one."""
    from haphic_b200._lib import HHError
    lg, T = 5, 16_000_000
    partitioned(lg)
    pcap, scap = region_cap(T, 1 << lg), spill_cap([T])
    pairs, parts = pick_pairs(w, lg, 1, seed=7)
    hot = hot_records(w, pairs, [pcap + scap + over], seed=8, grouped=False)
    rec = planted_stream(background(w, T - len(hot), parts, lg), hot, seed=9)
    pl = plan(w, rec, [(0, T)], lg)
    report("spill list boundary +{}".format(over), pl)
    assert pl["spill"] == scap + over and pl["spill_cap"] == scap
    tab = count(ctx, w, rec)
    if over:
        with pytest.raises(HHError, match="error 3: .*HH_LINKS_PARTITION=0"):
            tab.finish()
        tab.close()
    else:
        oracle_check(tab, w, rec)
        tab.close()


@pytest.mark.parametrize("calls", ["one", "split"])
def test_spill_across_partition_sets(ctx, w, partitioned, calls):
    """16M records, one pair planted 5.5M times, 32 partitions, sent in one call or as 1,000 records and then the rest.
    The second call opens a partition set of its own; its spill must fit as the one call's does.  The hot pair's first
    records sit in the regions of the first set and the rest spill from the second; a second hot pair spills too."""
    lg, T, first = 5, 16_000_000, 1000
    partitioned(lg)
    pairs, parts = pick_pairs(w, lg, 2, seed=10)
    hot = hot_records(w, pairs, [5_500_000, 1_000_000], seed=11, grouped=False)
    rec = planted_stream(background(w, T - len(hot)), hot, seed=12)
    cuts = [(0, T)] if calls == "one" else [(0, first), (first, T)]
    pl = plan(w, rec, cuts, lg)
    report("spill across partition sets, " + calls, pl)
    assert pl["spill_cap"] == spill_cap([T]) and pl["spill"] <= pl["spill_cap"]
    if calls == "split":
        s0, s1 = pl["sets"]
        hot_p = int(partition_of(hot[:1], w["rank"], w["n"], lg)[0])
        assert (s0["sized"], s1["sized"], s1["pcap"]) == (first, T - first, 754_049)
        assert 0 < s0["fill"][hot_p] <= s0["pcap"] and s1["fill"][hot_p] > 6 * s1["pcap"]
        # more than a spill list sized for the first call alone holds
        assert pl["spill"] > spill_cap([first])
    ref = oracle_check(count(ctx, w, rec, cuts), w, rec)
    assert len(ref["full_vals"]) > 0


def test_over_capacity_fails_clearly_and_direct_counts_it(ctx, w, monkeypatch):
    """One pair owns 75 % of 16M records: the spill list cannot hold the excess.  finish() says so and points to the
    direct engine; the table closes, a new one on the same context works, and the direct engine counts the stream."""
    from haphic_b200._lib import HHError
    T = 16_000_000
    monkeypatch.setenv("HH_LINKS_PARTITION", "1")
    monkeypatch.delenv("HH_LINKS_NPART_LOG", raising=False)
    pairs, _ = pick_pairs(w, default_npart_log(T), 1, seed=13)
    hot = hot_records(w, pairs, [12_000_000], seed=14, grouped=False)
    rec = planted_stream(background(w, T - len(hot)), hot, seed=15)
    pl = plan(w, rec, [(0, T)], default_npart_log(T))
    report("over capacity", pl)
    assert pl["spill"] > pl["spill_cap"]
    tab = count(ctx, w, rec)
    with pytest.raises(HHError, match="error 3: .*HH_LINKS_PARTITION=0"):
        tab.finish()
    tab.close()
    monkeypatch.setenv("HH_LINKS_PARTITION", "0")
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    tab.close()


# ---- host staging, partition counts, engine choice --------------------------------------------------------------------

@pytest.mark.parametrize("host", ["numpy", "pinned"])
def test_host_staging_reuses_both_buffers(ctx, w, counting_mode, host):
    """17M host records (three 8 Mi staging chunks: both buffers, one of them twice), then a second call of 7M records
    whose chunks wait on the events the first call left on both buffers."""
    rec = w["pool"][:24_000_000]
    cuts = [(0, 17_000_000), (17_000_000, 24_000_000)]
    tab = count(ctx, w, rec, cuts, host=host)
    oracle_check(tab, w, rec)
    tab.close()


@pytest.mark.parametrize("env_lg,lg", [(1, 1), (10, 10), (0, 1), (11, 10)])
def test_partition_count_extremes(ctx, w, partitioned, env_lg, lg):
    """HH_LINKS_NPART_LOG 1 and 10 (2 and 1024 partitions, the size of the scatter kernel's shared arrays), and 0 / 11
    clamped to them, each with a spilling partition (in the upper half of the partitions)."""
    T = 4_000_000
    partitioned(env_lg)
    pcap = region_cap(T, 1 << lg)
    pairs, parts = pick_pairs(w, lg, 1, seed=16, upper_first=True)
    n_hot = pcap + 20_000 if lg == 1 else 4 * pcap
    hot = hot_records(w, pairs, [n_hot], seed=17, grouped=False)
    rec = planted_stream(background(w, T - len(hot), parts, lg), hot, seed=18)
    pl = plan(w, rec, [(0, T)], lg)
    report("HH_LINKS_NPART_LOG={}".format(env_lg), pl)
    assert pl["sets"][0]["fill"][parts[0]] == n_hot and parts[0] >= (1 << lg) // 2
    assert 0 < pl["spill"] <= pl["spill_cap"] and np.delete(pl["sets"][0]["fill"], parts).max() <= pcap
    tab = count(ctx, w, rec)
    oracle_check(tab, w, rec)
    tab.close()


@pytest.mark.parametrize("n_rec", [(16 << 20) - 1, 16 << 20])
@pytest.mark.parametrize("n_ctg", [2047, 2048])
def test_default_engine_choice_at_its_thresholds(ctx, monkeypatch, n_rec, n_ctg):
    """Streams of at least 16 Mi records in one call over at least 2048 contigs are counted partitioned, the others
    directly; both exact.  A partitioned table refuses hh_links_merge (HH_ERR_STATE), a direct one accepts it."""
    from haphic_b200 import synth
    from haphic_b200._lib import HHError
    from haphic_b200.links import LinkTable, name_rank
    monkeypatch.delenv("HH_LINKS_PARTITION", raising=False)
    monkeypatch.delenv("HH_LINKS_NPART_LOG", raising=False)
    asm = synth.make_assembly(1, n_ctg, 20000, seed=19)
    assert asm.n == n_ctg
    rank, in_nx = name_rank(asm.names), np.ones(n_ctg, np.uint8)
    rec = synth.make_pairs(asm, 16 << 20, seed=20, device="cuda")[:n_rec].contiguous()
    tab = LinkTable(ctx, asm.lengths, rank, in_nx, FLANK_BP)
    tab.add(rec)            # one device call; unlike the asynchronous add it grows a direct table without a capacity hint
    none = torch.empty((0, 9), dtype=torch.int32, device="cuda")
    zero = torch.zeros(n_ctg, dtype=torch.int64, device="cuda")
    want_partitioned = n_rec >= (16 << 20) and n_ctg >= 2048
    print("\n{} records, {} contigs: {}".format(n_rec, n_ctg, "partitioned" if want_partitioned else "direct"))
    if want_partitioned:
        with pytest.raises(HHError, match="error 5"):
            tab.merge(none, zero, 0, 0)
    else:
        tab.merge(none, zero, 0, 0)
    info = tab.finish()
    assert info.n_records == n_rec
    assert_equals_oracle(tab, info, rec.cpu().numpy(), asm.lengths, rank, in_nx, FLANK_BP)
    tab.close()


# ---- stream indices at and above 2^31 ---------------------------------------------------------------------------------

@pytest.mark.parametrize("where", ["straddle_2_31", "top"])
def test_stream_offsets(ctx, w, counting_mode, where):
    """3M records (a planted pair that spills in the partitioned mode) streamed from an offset: across 2^31, and ending
    at the last index the API accepts (offset + n = 0xFFFFFFFE).  Pairs first seen at index 2^31 and at that last index
    are planted.  Dict order, first indices, the linked index and the matrix must all hold.
    The top run makes hh_links_finish / links_order_list allocate an order array of 4 * stream_end bytes, about 17 GB of
    device memory."""
    from oracle import haphic_oracle as orc
    T, lg = 3_000_000, 5
    pcap = region_cap(T, 1 << lg)
    offset = (1 << 31) - T // 2 if where == "straddle_2_31" else 0xFFFFFFFE - T
    pairs, _ = pick_pairs(w, lg, 1, seed=21)
    hot = hot_records(w, pairs, [4 * pcap], seed=22, grouped=False)
    rec = planted_stream(background(w, T - len(hot)), hot, seed=23)
    # two pairs of contigs on different chromosomes that the stream does not hold otherwise, both ends at flank positions
    seen = set((np.minimum(rec[:, 0], rec[:, 2]).astype(np.int64) * w["n"] + np.maximum(rec[:, 0], rec[:, 2])).tolist())
    rng = np.random.default_rng(24)
    fresh = []
    while len(fresh) < 2:
        a, b = (int(x) for x in rng.choice(w["eligible"], 2, replace=False))
        if w["asm"].chrom[a] != w["asm"].chrom[b] and min(a, b) * w["n"] + max(a, b) not in seen and (a, b) not in fresh:
            fresh.append((a, b))
    at = [(1 << 31) - offset if where == "straddle_2_31" else T // 2, T - 1]
    for (a, b), k in zip(fresh, at):
        rec[k] = (a, 10, b, int(w["lengths"][b]) - 10)
    if counting_mode == "partitioned":
        pl = plan(w, rec, [(0, T)], lg)
        report("stream offset {} ({})".format(offset, where), pl)
        assert pl["spill"] > 0
    tab = count(ctx, w, rec, offset=offset)
    ref = oracle_check(tab, w, rec, offset=offset)
    got = tab.fetch()
    assert int(got["first_full"][-1]) == offset + T - 1 == int(got["first_flank"][-1])
    if where == "straddle_2_31":
        e = int(np.nonzero(got["first_full"] == (1 << 31))[0][0])
        assert int(got["first_flank"][e]) == 1 << 31
    # linked index and matrix, a tenth of the contigs filtered out
    keep = (np.arange(w["n"]) % 10 != 3).astype(np.uint8)
    index, n_linked = tab.linked_index(keep)
    tail = np.nonzero((index < 0) & (keep > 0))[0].astype(np.int32)
    link, oindex = orc.dict_to_matrix(ref["flank_keys"], ref["flank_vals"], keep, tail_order=tail.tolist())
    assert n_linked == int((oindex >= 0).sum()) - len(tail)
    assert np.array_equal(np.where(index >= 0, index, oindex), oindex)
    mat = tab.to_matrix(keep, tail)
    m = mat.to_scipy()
    assert np.array_equal(m.indptr, link.indptr) and np.array_equal(m.indices, link.indices) and np.array_equal(m.data, link.data)
    mat.close()
    tab.close()


def test_stream_index_overflow_is_refused(ctx, w):
    """offset + n = 0xFFFFFFFF would give a record the index of the 'none' sentinel: add (host and device), the
    asynchronous add and route refuse it with HH_ERR_UNSUPPORTED."""
    from haphic_b200._lib import HHError
    from haphic_b200.links import LinkTable
    rec = np.ascontiguousarray(w["pool"][:16])
    off = 0xFFFFFFFF - len(rec)
    tab = LinkTable(ctx, w["lengths"], w["rank"], w["in_nx"], FLANK_BP)
    dev = torch.from_numpy(rec).cuda()
    for call in (lambda: tab.add(rec, stream_offset=off), lambda: tab.add(dev, stream_offset=off),
                 lambda: tab.add(dev, stream_offset=off, asynchronous=True), lambda: tab.route(dev, off, 2)):
        with pytest.raises(HHError, match="error 6"):
            call()
    tab.add(dev, stream_offset=off - 1)
    oracle_check(tab, w, rec, offset=off - 1)
    tab.close()
