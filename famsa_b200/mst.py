"""Host logic for a parallel replacement of MST-Prim's sequential vertex loop (reference src/tree/MSTPrim.cpp:280-549).

The reference relaxes and elects with the pair  (distance, ~ids_to_uint64(min id, max id))  compared
lexicographically (MSTPrim.cpp:366-386, 492-503).  The second component is unique per edge, so the pairs are a STRICT
TOTAL ORDER on the edges and the minimum spanning tree under it is unique -- whatever algorithm finds it.  Prim's
contribution beyond the edge set is only the order in which the vertices are visited from vertex 0 (mst_to_dendogram
needs it, MSTPrim.cpp:784-833), and that order can be replayed on the n-1 tree edges alone: at every step Prim takes
the smallest edge leaving the visited set, which is a tree edge (cut property), hence the smallest TREE edge leaving it.

So a device may find the MST with any parallel scheme (Boruvka: log2 n rounds of "every component picks its smallest
outgoing edge", each round one streaming pass over the distance triangle) and the host replays the visiting order in
O(n log n).  Precondition: distances must not depend on which endpoint is the row -- true for every pair except the
sequences of the reference's dropped-carry corner (64 identical residues on a word boundary); sets that contain such a
sequence keep the sequential loop (famsa_lcs_prim).

This module holds the host pieces (edge order, Prim-order replay, SLINK's labelling of the same MST) and a reference
Kruskal used by the tests; the device side is famsa_lcs_prim / famsa_lcs_slink (DESIGN.md section 6).
"""
from __future__ import annotations

import heapq

import numpy as np

_FULL = 0xFFFFFFFFFFFFFFFF


def edge_key(a: int, b: int) -> int:
    """~ids_to_uint64(min, max) as the reference packs it (MSTPrim.h:432-439)."""
    lo, hi = (a, b) if a < b else (b, a)
    return _FULL ^ ((lo << 32) + hi)


def kruskal_total_order(n: int, tri: np.ndarray) -> list[tuple[int, int, float]]:
    """The unique MST under the (distance, key) order.  tri: packed lower triangle of float64 distances,
    entry (i, j), i > j, at i*(i-1)/2 + j.  Returns n-1 edges (from < to, dist).  O(n^2 log n): test-sized inputs."""
    ii, jj = np.tril_indices(n, -1)
    keys = np.array([edge_key(int(a), int(b)) for a, b in zip(jj, ii)], dtype=np.uint64)
    order = np.lexsort((keys, tri))                     # primary: distance, secondary: key
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    out = []
    for e in order:
        a, b = int(jj[e]), int(ii[e])
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
            out.append((a, b, float(tri[e])))
            if len(out) == n - 1:
                break
    return out


def slink_tree(n: int, edges) -> np.ndarray:
    """SingleLinkage<>::run's tree (SingleLinkage.cpp:30-189) from the MST of its distances.  With SLINK_HANDLE_TIES the
    reference orders distances by (distance, ids_to_uint64 descending) -- the order above -- so its hierarchy is that
    MST merged in Kruskal order, and its relabelling (stable_sort of lambda, then index[pi[j]] = n + k) names a merge
    by the largest member of each side: for the edge joining clusters with largest members a < b, emit
    (node(a), node(b)); the merged cluster becomes node n + k, keyed by b.  edges: n-1 (from, to, dist) in any order.
    Returns the n-1 merges, (n-1, 2) int32.  famsa_b200/csrc/tree.cu slink_labels is the same code in C++."""
    order = sorted(edges, key=lambda e: (e[2], edge_key(e[0], e[1])))
    parent = list(range(n))
    top = list(range(n))                                # largest member of the cluster rooted here
    node = list(range(n))                               # current node id of the cluster keyed by a member

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    out = np.zeros((max(n - 1, 0), 2), dtype=np.int32)
    for k, (a, b, _) in enumerate(order):
        ra, rb = find(int(a)), find(int(b))
        lo, hi = sorted((top[ra], top[rb]))
        out[k] = node[lo], node[hi]
        node[hi] = n + k
        parent[ra] = rb
        top[rb] = hi
    return out


def prim_replay(n: int, edges) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Visiting order of Prim from vertex 0 on a spanning tree given as (from, to, dist) edges.  Returns
    (edge_from, edge_to, edge_dist, prim_order) exactly as famsa_lcs_prim does: edge k was added with the (k+1)-th
    vertex, edge_from < edge_to, prim_order[i] = visiting position of vertex i."""
    adj = [[] for _ in range(n)]
    for a, b, d in edges:
        adj[a].append((d, edge_key(a, b), b))
        adj[b].append((d, edge_key(a, b), a))
    order = np.full(n, n, dtype=np.int32)
    order[0] = 0
    heap = list(adj[0])
    heapq.heapify(heap)
    ef, et, ed = [], [], []
    step = 0
    while heap:
        d, k, v = heapq.heappop(heap)
        if order[v] != n:
            continue
        step += 1
        order[v] = step
        p = _FULL ^ k
        ef.append(p >> 32); et.append(p & 0xFFFFFFFF); ed.append(d)
        for e in adj[v]:
            if order[e[2]] == n:
                heapq.heappush(heap, e)
    return np.array(ef, np.int32), np.array(et, np.int32), np.array(ed, np.float64), order
