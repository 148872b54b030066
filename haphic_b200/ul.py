"""Ultra-long read contig paths for `haphic cluster --ul` (scripts/HapHiC_cluster.py:1755-1985 of the reference).

The UL BAM is read once by the native reader (hh_ul_* in libhaphic_b200.so): it applies the alignment filters and the
primary / supplementary state machine and returns the header's references and one link event per accepted alignment
pair.  Here the events become the reference's weighted semi-contig graph (networkx, same edge-insertion order), which is
pruned and cut into contig paths exactly as parse_ul_alignments does.  The paths then act in three places:

* ``whitelist`` -- the contigs of the inter-contig steps, kept through the fragment filters;
* the HT and full links of every adjacent contig pair on a path count twice: on the host dicts
  (add_HT_links_based_on_ul / add_flank_and_full_links_based_on_ul) or, on the array path, when the device table is
  fetched (LinkTable.set_ul_pairs);
* the flank links between two different contigs of one path count twice: on the host dict, or inside the device matrix
  (``ul_path`` / ``ul_parent`` per table fragment, LinkTable.to_matrix).
"""

from __future__ import annotations

import ctypes as C
import os
from itertools import combinations

import numpy as np


def _contig(node):
    return node.rsplit("_", 1)[0]


def read_ul_events(path, args):
    """(reference names, reference lengths, events int32 [n, 4]) of the native reader (hh_ul_open): left and right
    semi-contig (2 * reference + 0 for `_H`, 1 for `_T`), primary and supplementary reference, in file order."""
    from ._lib import check, load
    lib = load()
    h = C.c_void_p()
    check(lib.hh_ul_open(os.fsencode(path), int(args.threads), int(args.min_ul_mapq), int(args.min_ul_alignment_length),
                         int(args.max_distance_to_end), float(args.max_overlap_ratio), int(args.max_gap_len), C.byref(h)))
    try:
        n_ref, nbytes, n_ev, n_rec = C.c_int32(), C.c_int64(), C.c_int64(), C.c_int64()
        check(lib.hh_ul_info(h, C.byref(n_ref), C.byref(nbytes), C.byref(n_ev), C.byref(n_rec)))
        names = C.create_string_buffer(max(1, nbytes.value))
        ref_len = np.empty(n_ref.value, np.int64)
        events = np.empty((n_ev.value, 4), np.int32)
        check(lib.hh_ul_fetch(h, names, ref_len.ctypes.data_as(C.c_void_p), events.ctypes.data_as(C.c_void_p)))
    finally:
        lib.hh_ul_close(h)
    ref_names = names.raw[:nbytes.value].split(b"\x00")[:-1] if nbytes.value else []
    return [n.decode() for n in ref_names], ref_len, events


def _bump(graph, a, b):
    if graph.has_edge(a, b):
        graph[a][b]["weight"] += 1
    else:
        graph.add_edge(a, b, weight=1)


def event_graph(ref_names, events):
    """The semi-contig graph of parse_supplementary_aln_list (1795-1810): per event the inter-contig edge, then the `_H`-`_T`
    edges of the primary's and of the supplementary's contig, each adding 1 to a weight."""
    from networkx import Graph
    semi = ("_H", "_T")
    graph = Graph()
    for left, right, prim, supp in events.tolist():
        _bump(graph, ref_names[left >> 1] + semi[left & 1], ref_names[right >> 1] + semi[right & 1])
        _bump(graph, ref_names[prim] + "_H", ref_names[prim] + "_T")
        _bump(graph, ref_names[supp] + "_H", ref_names[supp] + "_T")
    return graph


def extract_paths(graph, min_ul_support, ref_length, logger):
    """Contig paths of the pruned graph (1871-1907).  Every edge below ``min_ul_support`` goes (the reference compares
    whole node names there, so the `_H`-`_T` edges too); then every inter-contig edge at a node of degree > 2, degrees taken
    before any removal.  Components of >= 4 nodes are paths: a linear one runs between its two degree-1 nodes, a ring is
    cut at its lightest edge (the first of a stable sort by weight)."""
    from networkx import connected_components, shortest_path
    for a, b, d in list(graph.edges(data=True)):
        if d["weight"] < min_ul_support:
            graph.remove_edge(a, b)
    degree = dict(graph.degree())
    for a, b in list(graph.edges()):
        if (degree[a] > 2 or degree[b] > 2) and _contig(a) != _contig(b):
            graph.remove_edge(a, b)
    path_list = []
    for nodes in connected_components(graph):
        if len(nodes) < 4:
            continue
        logger.debug([(node, graph.degree(node)) for node in nodes])
        sub = graph.subgraph(nodes).copy()
        ends = [node for node in nodes if sub.degree(node) == 1]
        if len(ends) == 2:
            start, stop = ends
        else:
            start, stop, _w = sorted(((a, b, graph[a][b]["weight"]) for a, b in sub.edges()), key=lambda x: x[2])[0]
            sub.remove_edge(start, stop)
        path = shortest_path(sub, start, stop)
        path_list.append(path)
        logger.debug("{}\t{}".format("->".join(path), "-".join(str(ref_length[_contig(node)] // 2) for node in path)))
    return path_list


def parse_ul_alignments(args, logger):
    """path_list of the reference's parse_ul_alignments (1763-1909) for ``args.ul``."""
    logger.info("Parsing input ultra-long alignments...")
    ref_names, ref_len, events = read_ul_events(args.ul, args)
    ref_length = dict(zip(ref_names, ref_len.tolist()))
    return extract_paths(event_graph(ref_names, events), args.min_ul_support, ref_length, logger)


def linked_steps(path_list):
    """Per path, the inter-contig steps (path[i], path[i + 1]) at odd i (1915-1918)."""
    return [[(path[i], path[i + 1]) for i in range(1, len(path) - 1, 2)] for path in path_list]


def whitelist(path_list):
    """Contigs of the inter-contig steps (run(), 2813-2824)."""
    return {_contig(node) for steps in linked_steps(path_list) for step in steps for node in step}


def adjacent_pairs(path_list):
    """[(ctg1, ctg2, node1, node2)] per inter-contig step, ordered by contig name as the reference's dict keys are."""
    out = []
    for steps in linked_steps(path_list):
        for a, b in steps:
            (c1, n1), (c2, n2) = sorted(((_contig(a), a), (_contig(b), b)))
            out.append((c1, c2, n1, n2))
    return out


def path_sets(path_list):
    """Per path, the set of contigs of its inter-contig steps (ul_linked_ctgs of 1938-1950)."""
    return [{_contig(node) for step in steps for node in step} for steps in linked_steps(path_list)]


def add_HT_links_based_on_ul(path_list, HT_link_dict, logger):
    """1912-1933: the HT link of every adjacent pair's joined semi-contigs counts twice, with the reference's debug lines.
    ``HT_link_dict`` is the host dict (doubled here) or, on the array path, the set of those keys that the device table
    holds (present_keys; the table doubles them when it is fetched), which only logs."""
    for _c1, _c2, n1, n2 in adjacent_pairs(path_list):
        if (n1, n2) in HT_link_dict:
            logger.debug("update HT_link_dict: {} {}".format(n1, n2))
            if isinstance(HT_link_dict, dict):
                HT_link_dict[(n1, n2)] *= 2
        else:
            logger.debug("{} {} not in HT_link_dict".format(n1, n2))


def add_flank_and_full_links_based_on_ul(path_list, flank_link_dict, full_link_dict, bin_set, logger):
    """1936-1985: the full links of every adjacent pair and the flank links between any two different contigs of one path
    (bins by their contig) count twice.  On the host dicts both are doubled here; on the array path ``full_link_dict`` is
    the set of the adjacent pairs that the device table holds (present_keys) and ``flank_link_dict`` None: the device
    doubles both (fetch, matrix kernels) and this only logs the reference's debug lines.  The reference also prints every
    doubled flank entry to stdout; that print is not reproduced."""
    for c1, c2, n1, n2 in adjacent_pairs(path_list):
        if (c1, c2) in full_link_dict:
            logger.debug("update full_link_dict: {} {}".format(c1, c2))
            if isinstance(full_link_dict, dict):
                full_link_dict[(c1, c2)] *= 2
        else:
            logger.debug("{} {} not in full_link_dict".format(n1, n2))
    if flank_link_dict is None:
        return
    joined = set()
    for ctgs in path_sets(path_list):
        for a, b in combinations(ctgs, 2):
            joined.add((a, b))
            joined.add((b, a))
    if not joined:
        return
    for fi, fj in flank_link_dict:
        ci = fi.rsplit("_bin", 1)[0] if fi in bin_set else fi
        cj = fj.rsplit("_bin", 1)[0] if fj in bin_set else fj
        if (ci, cj) in joined:
            flank_link_dict[(fi, fj)] *= 2


def fragment_arrays(path_list, contig_names, frag_parent):
    """(ul_path, ul_parent) int32 per table fragment for the device matrix: the id of the path whose contigs include the
    fragment's contig (-1 = none), and that contig's id (``frag_parent``, an index into ``contig_names``)."""
    path_of = {c: k for k, ctgs in enumerate(path_sets(path_list)) for c in ctgs}
    ctg_path = np.fromiter((path_of.get(n, -1) for n in contig_names), dtype=np.int32, count=len(contig_names))
    parent = np.ascontiguousarray(frag_parent, dtype=np.int32)
    return ctg_path[parent], parent


def table_pairs(path_list, names):
    """(key_i, key_j, ht_slot) int32 of the adjacent pairs whose two contigs are in ``names`` (contig ids, name(key_i) <
    name(key_j)); ht_slot = 2 * ti + tj of the joined semi-contigs (hh_links_set_ul_pairs)."""
    ids = {n: k for k, n in enumerate(names)}
    ki, kj, slot = [], [], []
    for c1, c2, n1, n2 in adjacent_pairs(path_list):
        if c1 == c2 or c1 not in ids or c2 not in ids:
            continue
        ki.append(ids[c1])
        kj.append(ids[c2])
        slot.append(2 * (n1[-1] == "T") + (n2[-1] == "T"))
    return np.asarray(ki, np.int32), np.asarray(kj, np.int32), np.asarray(slot, np.int32)


def present_keys(path_list, names, key_i, key_j, ht):
    """(HT keys, full keys) of the adjacent pairs that the fetched contig-level table holds: the HT_link_dict keys
    (node1, node2) with a non-zero count and the full_link_dict keys (ctg1, ctg2).  For the debug lines of the array path."""
    ids = {n: k for k, n in enumerate(names)}
    n = len(names)
    table_keys = key_i.astype(np.int64) * n + key_j.astype(np.int64)
    pairs = [(c1, c2, n1, n2) for c1, c2, n1, n2 in adjacent_pairs(path_list) if c1 in ids and c2 in ids]
    want = np.array([ids[c1] * n + ids[c2] for c1, c2, _n1, _n2 in pairs], np.int64)
    order = np.argsort(table_keys, kind="stable")
    pos = np.searchsorted(table_keys[order], want)
    ht_keys, full_keys = set(), set()
    for (c1, c2, n1, n2), p in zip(pairs, pos.tolist()):
        if p < len(order) and table_keys[order[p]] == ids[c1] * n + ids[c2]:
            e = int(order[p])
            full_keys.add((c1, c2))
            if ht[e, 2 * (n1[-1] == "T") + (n2[-1] == "T")]:
                ht_keys.add((n1, n2))
    return ht_keys, full_keys
