"""Seeded synthetic workloads with the shapes of the reference's datasets (no downloads; the real loaders
dataset/metr_la.py, pems_bay.py need the network).  Recipes from SURVEY.md section 8(d)."""
import numpy as np


def random_digraph(num_nodes: int, num_pairs: int, self_loops: bool, seed: int = 0, weight_low=0.1, weight_high=1.0):
    """`num_pairs` distinct directed off-diagonal edges (uniform, without replacement) + optional self
    loops (w=1); edge list in ROW-MAJOR order (= dense_to_sparse of the adjacency, metr_la.py:92)."""
    rng = np.random.RandomState(seed)
    n = num_nodes
    off = np.flatnonzero(~np.eye(n, dtype=bool).ravel())
    pick = rng.choice(off, size=num_pairs, replace=False)
    A = np.zeros(n * n, dtype=np.float32)
    A[pick] = rng.uniform(weight_low, weight_high, size=num_pairs).astype(np.float32)
    A = A.reshape(n, n)
    if self_loops:
        A[np.arange(n), np.arange(n)] = 1.0
    row, col = np.nonzero(A)
    return np.stack([row, col]).astype(np.int64), A[row, col].astype(np.float32)


def metr_la_like(seed: int = 0, t_total: int = 2048):
    """N=207, E=1722 (207 loops + 1515 pairs), F=2, z-scored-like N(0,1) series (t_total,207,2)."""
    ei, ew = random_digraph(207, 1515, True, seed)
    rng = np.random.RandomState(seed + 1)
    return ei, ew, rng.standard_normal((t_total, 207, 2)).astype(np.float32)


def pems_bay_like(seed: int = 0, t_total: int = 2048):
    """N=325, E=2694 (325 loops + 2369 pairs), F=2."""
    ei, ew = random_digraph(325, 2369, True, seed)
    rng = np.random.RandomState(seed + 1)
    return ei, ew, rng.standard_normal((t_total, 325, 2)).astype(np.float32)


def _undirected_links(n: int, links: int, seed: int):
    """`links` distinct undirected links between n nodes (uniform, without replacement), both directions, no loops, unweighted;
    edge list in ROW-MAJOR order."""
    rng = np.random.RandomState(seed)
    iu = np.stack(np.triu_indices(n, 1), axis=1)
    pick = iu[rng.choice(len(iu), size=links, replace=False)]
    A = np.zeros((n, n), dtype=np.float32)
    A[pick[:, 0], pick[:, 1]] = 1
    A[pick[:, 1], pick[:, 0]] = 1
    row, col = np.nonzero(A)
    return np.stack([row, col]).astype(np.int64)


def pems04_like(seed: int = 0):
    """N=307, 340 undirected links (E=680, symmetric, no loops), unweighted."""
    return _undirected_links(307, 340, seed)


def pems03_like(seed: int = 0):
    """N=358, 547 undirected links (E=1094, symmetric, no loops), unweighted: the PeMS03 sensor network's shape."""
    return _undirected_links(358, 547, seed)


def pems07_like(seed: int = 0):
    """N=883, 866 undirected links (E=1732, symmetric, no loops), unweighted: the PeMS07 sensor network's shape."""
    return _undirected_links(883, 866, seed)


def large_graph(num_nodes=10000, num_edges=100000, seed=0):
    """cfg5: random directed non-loop edges, w~U(0.1,1)."""
    rng = np.random.RandomState(seed)
    keys = set()
    while len(keys) < num_edges:
        r = rng.randint(0, num_nodes, size=num_edges)
        c = rng.randint(0, num_nodes, size=num_edges)
        for a, b in zip(r, c):
            if a != b:
                keys.add(int(a) * num_nodes + int(b))
                if len(keys) == num_edges:
                    break
    k = np.array(sorted(keys), dtype=np.int64)
    ei = np.stack([k // num_nodes, k % num_nodes]).astype(np.int64)
    ew = rng.uniform(0.1, 1.0, size=num_edges).astype(np.float32)
    return ei, ew


def banded_graph(num_nodes=10000, num_edges=100000, span=64, seed=0):
    """Sensor-network-like graph: nodes numbered along the roads, every edge joins two nodes at most `span` apart (the kNN-by-road-distance
    adjacency of METR-LA / PEMS-BAY after a locality-preserving ordering); directed, no loops, w~U(0.1,1)."""
    rng = np.random.RandomState(seed)
    keys = set()
    while len(keys) < num_edges:
        r = rng.randint(0, num_nodes, size=num_edges)
        d = rng.randint(1, span + 1, size=num_edges) * rng.choice([-1, 1], size=num_edges)
        c = r + d
        ok = (c >= 0) & (c < num_nodes)
        for a, b in zip(r[ok], c[ok]):
            keys.add(int(a) * num_nodes + int(b))
            if len(keys) == num_edges:
                break
    k = np.array(sorted(keys), dtype=np.int64)
    ei = np.stack([k // num_nodes, k % num_nodes]).astype(np.int64)
    ew = rng.uniform(0.1, 1.0, size=num_edges).astype(np.float32)
    return ei, ew
