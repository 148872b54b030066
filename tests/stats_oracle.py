"""Host reference of the reassignment statistics of `haphic cluster` (output_statistics, scripts/HapHiC_cluster.py v1.0.7,
2245-2478) and of the full-link phasing reduction, for the tests to compare the device against:

  * the reference's dict walk restated literally (parse_link_dict, cal_link_density and the per-contig loop, 2355-2391);
  * the same ranking and statistics on arrays in numpy (exact fp64 arithmetic in the reference's order, at sizes the dict
    walk cannot reach), checked against the dict walk themselves;
  * reduce_inter_hap_HiC_links (695-707) on the arrays of a LinkArrays."""

import sys
from collections import defaultdict

import numpy as np


# ------------------------------------------------------------------------------------------------
# the reference's dict walk
# ------------------------------------------------------------------------------------------------

def parse_link_dict(link_dict, ctg_group_dict):
    """{contig: {group: links}} (2252-2268): both ends of every entry in insertion order, groups in the order first met; a
    group's first link is stored as it is, the later ones are added to it."""
    out = defaultdict(dict)
    for (ci, cj), links in link_dict.items():
        gi, gj = ctg_group_dict[ci], ctg_group_dict[cj]
        for ctg, grp in ((ci, gj), (cj, gi)):
            if grp != "ungrouped":
                if grp in out[ctg]:
                    out[ctg][grp] += links
                else:
                    out[ctg][grp] = links
    return out


def cal_link_density(max_group, current_group, max_links, group_RE_sites, ctg_RE_sites):
    if max_group == current_group:
        return max_links / group_RE_sites
    return max_links / (group_RE_sites + ctg_RE_sites - 1)


def ranked_from_dict(link_dict, ctg_group):
    """{contig: [(group, links), ...]} ranked as 2365 sorts them: links descending, ties in first-met order."""
    return {ctg: sorted(groups.items(), key=lambda x: x[1], reverse=True)
            for ctg, groups in parse_link_dict(link_dict, ctg_group).items()}


def statistics_from_dict(fa_dict, link_dict, ctg_group, group_RE):
    """The three per-contig lists of output_statistics, the reference's loop over fa_dict (2355-2391)."""
    group_links = parse_link_dict(link_dict, ctg_group)
    best_links, best_density, best_ratio = [], [], []
    for ctg in fa_dict:
        if ctg not in group_links:
            best_links.append((ctg, 0))
            best_density.append((ctg, 0))
            best_ratio.append((ctg, 0))
            continue
        ranked = sorted(group_links[ctg].items(), key=lambda x: x[1], reverse=True)
        top_group, top_links = ranked[0]
        cur = ctg_group[ctg]
        ctg_RE = fa_dict[ctg][2]
        dens = cal_link_density(top_group, cur, top_links, group_RE[top_group], ctg_RE)
        if len(group_RE) > 1:
            others = sum([cal_link_density(g, cur, v, group_RE[g], ctg_RE) for g, v in ranked[1:]]) / (len(group_RE) - 1)
        else:
            others = 0
        best_links.append((ctg, top_links))
        best_density.append((ctg, dens))
        best_ratio.append((ctg, dens / others if others else 1000000))
    return best_links, best_density, best_ratio


# ------------------------------------------------------------------------------------------------
# the same on arrays
# ------------------------------------------------------------------------------------------------

def python_numbers(sums, is_float):
    """Sums as the reference's dict values: ints, or floats where any contributing link was a float."""
    if is_float is None:
        return sums.tolist()
    return [v if f else int(v) for v, f in zip(sums.tolist(), is_float.tolist())]


def ranked_group_links(links, gid, ng):
    """(contig, group, links, is_float) of parse_link_dict's sums over a LinkArrays, ordered by (contig, rank); gid[c] = group
    of contig c (-1 = ungrouped), ng > every group.  parse_link_dict adds a contig's links to one group one by one in its
    visiting order (first end of entry 0, second end of entry 0, first end of entry 1, ...): integer prefixes are exact in
    fp64, so plain sequential fp64 adds in that order give its sums, and a sum is a float iff one of its links is.  Integer
    links (is_float None) are summed as int64 and is_float comes back None.  The adds run position by position across all
    (contig, group) segments at once, longest segments first, so every step works on a prefix of the segments."""
    m = len(links)
    ctg = np.empty(2 * m, np.int64)
    oth = np.empty(2 * m, np.int64)
    ctg[0::2], ctg[1::2] = links.key_i, links.key_j
    oth[0::2], oth[1::2] = links.key_j, links.key_i
    g = gid[oth]
    pos = np.nonzero(g >= 0)[0]                                 # position in the visiting order
    if len(pos) == 0:
        z = np.zeros(0, np.int64)
        return z, z, np.zeros(0, links.values.dtype), None if links.is_float is None else np.zeros(0, bool)
    key = ctg[pos] * ng + g[pos]
    order = np.argsort(key, kind="stable")                     # by key, then by position
    ks = key[order]
    val = np.repeat(links.values, 2)[pos][order]
    starts = np.concatenate([[0], np.nonzero(np.diff(ks))[0] + 1])
    seg_len = np.diff(np.concatenate([starts, [len(ks)]]))
    by_len = np.argsort(-seg_len, kind="stable")
    st_sorted, len_sorted = starts[by_len], seg_len[by_len]
    acc = np.zeros(len(starts), val.dtype)
    for p in range(int(len_sorted[0])):
        k = int(np.searchsorted(-len_sorted, -p, side="left"))   # segments longer than p: a prefix
        acc[:k] += val[st_sorted[:k] + p]
    sums = np.empty(len(starts), val.dtype)
    sums[by_len] = acc
    is_f = None
    if links.is_float is not None:
        is_f = np.logical_or.reduceat(np.repeat(links.is_float, 2)[pos][order], starts)
    first = pos[order][starts]                                  # first position of each segment
    c_of, g_of = ks[starts] // ng, ks[starts] % ng
    rank = np.lexsort((first, -sums, c_of))
    return c_of[rank], g_of[rank], sums[rank], None if is_f is None else is_f[rank]


def group_ids(names, ctg_group):
    """gid[c] of every contig (-1 = ungrouped) and the number of groups it implies."""
    gid = np.array([-1 if ctg_group[nm] == "ungrouped" else ctg_group[nm] for nm in names], dtype=np.int64)
    return gid, int(gid.max()) + 1


def ranked_lists(names, c_of, g_of, sums, is_float=None):
    """{contig: [(group, links), ...]} from arrays ordered by (contig, rank), the form ranked_from_dict gives."""
    out = {}
    if len(c_of) == 0:
        return out
    cuts = np.concatenate([[0], np.nonzero(np.diff(c_of))[0] + 1, [len(c_of)]])
    g_list, s_list = g_of.tolist(), python_numbers(sums, is_float)
    for k in range(len(cuts) - 1):
        lo, hi = int(cuts[k]), int(cuts[k + 1])
        out[names[int(c_of[lo])]] = list(zip(g_list[lo:hi], s_list[lo:hi]))
    return out


def best_group_statistics(fa_dict, links, ctg_group, group_RE):
    """statistics_from_dict on a LinkArrays, vectorised: same arithmetic in the same order.  int / int true divisions become
    fp64 divisions of the same integers (both correctly rounded), and the sum over ranked[1:] is accumulated position by
    position, left to right, like sum()."""
    names = links.names
    zero = [(ctg, 0) for ctg in fa_dict]
    gid, ng = group_ids(names, ctg_group)
    if len(links) == 0 or ng == 0:
        return zero, list(zero), list(zero)
    c_of, g_of, sums, is_float = ranked_group_links(links, gid, ng)
    if len(c_of) == 0:
        return zero, list(zero), list(zero)
    n_groups = len(group_RE)
    RE_g = np.array([group_RE[g] for g in range(ng)], dtype=np.int64)
    RE_c = np.array([fa_dict[nm][2] for nm in names], dtype=np.int64)
    starts = np.concatenate([[0], np.nonzero(np.diff(c_of))[0] + 1])
    seg_len = np.diff(np.concatenate([starts, [len(c_of)]]))
    seg_c = c_of[starts]
    denom = RE_g[g_of] + np.repeat(RE_c[seg_c] - 1, seg_len)              # cal_link_density: other group
    same = np.nonzero(g_of == np.repeat(gid[seg_c], seg_len))[0]          # ... the contig's own group
    denom[same] = RE_g[g_of[same]]
    dens = sums.astype(np.float64) / denom.astype(np.float64)
    # sum(): left to right; CPython >= 3.12 adds floats with Neumaier's compensated summation (bltinmodule.c), earlier
    # versions plainly
    acc = np.zeros(len(starts), np.float64)
    comp = np.zeros(len(starts), np.float64)
    neumaier = sys.version_info >= (3, 12)
    for pos in range(1, int(seg_len.max())):
        m = np.nonzero(seg_len > pos)[0]
        x = dens[starts[m] + pos]
        f = acc[m]
        t = f + x
        if neumaier:
            comp[m] += np.where(np.abs(f) >= np.abs(x), (f - t) + x, (x - t) + f)
        acc[m] = t
    if neumaier:
        fix = (comp != 0) & np.isfinite(comp)
        acc[fix] += comp[fix]
    others = acc / (n_groups - 1) if n_groups > 1 else np.zeros(len(starts))
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = dens[starts] / others
    has = {int(c): k for k, c in enumerate(seg_c.tolist())}
    top_links = python_numbers(sums[starts], None if is_float is None else is_float[starts])
    top_dens, others_l, ratio_l = dens[starts].tolist(), others.tolist(), ratio.tolist()
    name_idx = {nm: i for i, nm in enumerate(names)}
    best_links, best_density, best_ratio = [], [], []
    for ctg in fa_dict:
        k = has.get(name_idx.get(ctg, -1))
        if k is None:
            best_links.append((ctg, 0))
            best_density.append((ctg, 0))
            best_ratio.append((ctg, 0))
            continue
        best_links.append((ctg, top_links[k]))
        best_density.append((ctg, top_dens[k]))
        best_ratio.append((ctg, ratio_l[k] if others_l[k] else 1000000))
    return best_links, best_density, best_ratio


# ------------------------------------------------------------------------------------------------
# the phasing reduction of the full links
# ------------------------------------------------------------------------------------------------

def reduce_phasing(links, hap, phasing_weight):
    """reduce_inter_hap_HiC_links (695-707) on a LinkArrays, returned as a new one: entries between haplotypes (``hap`` per
    contig) become v - v * w in fp64 (two roundings, as Python evaluates it), zeros are dropped, the order is kept.  With
    w = 1 every such entry is dropped and the values stay integers."""
    inter = hap[links.key_i] != hap[links.key_j]
    if not inter.any():
        return links
    x = links.values.astype(np.float64)
    xi = x[inter]
    x[inter] = xi - xi * float(phasing_weight)
    keep = x != 0
    inter = inter[keep]
    if links.is_float is None and not inter.any():
        out = type(links)(links.names, links.key_i[keep], links.key_j[keep], links.values[keep])
    else:
        flt = inter if links.is_float is None else (links.is_float[keep] | inter)
        out = type(links)(links.names, links.key_i[keep], links.key_j[keep], x[keep], flt)
    out.phased = True
    return out
