"""The float64 Leiden restatement (tests/leiden_ref.py) that the device Leiden is tested against, checked without a GPU: its
quality is networkx's modularity, its communities are connected, it recovers a planted partition and it does not fall short of
networkx's Louvain."""
import networkx as nx
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph

from leiden_ref import canonical, leiden_ref, quality


def random_graph(n, p, seed):
    rng = np.random.default_rng(seed)
    U = sp.random(n, n, density=p, random_state=rng, data_rvs=lambda m: rng.uniform(0.05, 1.0, m))
    A = sp.triu(U, k=1)
    return sp.csr_matrix(A + A.T)


def planted(sizes, p_in, p_out, seed):
    g = nx.random_partition_graph(sizes, p_in, p_out, seed=seed)
    A = nx.to_scipy_sparse_array(g, nodelist=range(sum(sizes)), format="csr").astype(np.float64)
    truth = np.repeat(np.arange(len(sizes)), sizes)
    return sp.csr_matrix(A), truth


def as_nx(A):
    return nx.from_scipy_sparse_array(sp.csr_matrix(A))


def parts(labels):
    return [set(np.flatnonzero(labels == c).tolist()) for c in np.unique(labels)]


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("gamma", [0.4, 1.0, 2.5])
def test_quality_is_networkx_modularity(seed, gamma):
    A = random_graph(60, 0.1, seed)
    labels = np.random.default_rng(seed).integers(0, 5, 60)
    want = nx.community.modularity(as_nx(A), parts(labels), weight="weight", resolution=gamma)
    assert abs(quality(A, labels, gamma) - want) <= 1e-12


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("gamma", [0.4, 1.0])
def test_communities_are_connected(seed, gamma):
    A = random_graph(150, 0.03, seed)
    labels, _ = leiden_ref(A, gamma)
    for c in np.unique(labels):
        idx = np.flatnonzero(labels == c)
        assert csgraph.connected_components(A[idx][:, idx], directed=False)[0] == 1, c


def test_recovers_a_planted_partition():
    A, truth = planted([40, 30, 30, 20], 0.5, 0.005, seed=1)
    labels, _ = leiden_ref(A, 1.0)
    assert np.array_equal(labels, canonical(truth))


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("gamma", [0.4, 1.0])
def test_quality_matches_networkx_louvain(seed, gamma):
    A, _ = planted([50, 40, 30, 30, 20], 0.15, 0.02, seed=seed)
    labels, _ = leiden_ref(A, gamma)
    louvain = nx.community.louvain_communities(as_nx(A), weight="weight", resolution=gamma, seed=0)
    q_nx = nx.community.modularity(as_nx(A), louvain, weight="weight", resolution=gamma)
    assert quality(A, labels, gamma) >= q_nx - 0.005


def test_labels_are_canonical_and_iterations_stop():
    A = random_graph(120, 0.05, 7)
    labels, its = leiden_ref(A, 1.0)
    sizes = np.bincount(labels)
    assert np.all(np.diff(sizes) <= 0)
    assert np.array_equal(labels, canonical(labels))
    assert 1 <= its < 100
