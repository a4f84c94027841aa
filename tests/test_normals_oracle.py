"""Host tests of the normal-estimation oracle (tests/normals_oracle.py): its PCA against a direct solve, its forest
against scipy's minimum spanning tree and connected components, and its orientation on a sphere."""
import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components, minimum_spanning_tree

from tests.normals_oracle import canonical, graph_edges, knn_rows, orient, parent_edges, pca_normals


def _sphere(n, seed=0):
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(n, 3))
    return (p / np.linalg.norm(p, axis=1, keepdims=True)).astype(np.float32)


def _clusters(seed):
    """a few far-apart blobs of random points: a k-NN graph of several components"""
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.normal(size=(150, 3)) * 0.3 + c for c in ((0, 0, 0), (40, 0, 0), (0, 40, 5))]).astype(
        np.float32)


def test_canonical_sign():
    n = np.array([[-0.6, 0.8, 0.0], [0.0, 0.0, -1.0], [-0.5, 0.5, 0.1], [0.3, -0.3, 0.1]], np.float32)
    c = canonical(n)
    assert np.array_equal(c, np.array([[-0.6, 0.8, 0.0], [0.0, 0.0, 1.0], [0.5, -0.5, -0.1], [0.3, -0.3, 0.1]], np.float32))


def test_pca_plane_and_invalid_rows():
    rng = np.random.default_rng(1)
    p = np.concatenate([rng.uniform(-1, 1, (200, 2)), np.zeros((200, 1))], 1).astype(np.float32)
    idx = knn_rows(p, 8)
    n, lam = pca_normals(p, idx)
    assert np.allclose(n, [0, 0, 1], atol=1e-6)
    assert (lam[:, 0] < 1e-12).all()
    idx[3, 5] = -1
    n, _ = pca_normals(p, idx)
    assert np.isnan(n[3]).all() and np.isfinite(np.delete(n, 3, 0)).all()


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("k", [3, 8, 20])
def test_forest_matches_scipy(seed, k):
    p = _clusters(seed) if seed == 2 else np.random.default_rng(seed).uniform(-1, 1, (400, 3)).astype(np.float32)
    idx = knn_rows(p, k)
    n, _ = pca_normals(p, idx)
    res = orient(p, n, idx)
    lo, hi, w = graph_edges(n, idx)
    P = p.shape[0]
    # scipy drops zero weights: shift every weight by 1 (a uniform shift keeps the minimum spanning forest)
    g = coo_matrix((w.astype(np.float64) + 1.0, (lo, hi)), shape=(P, P)).tocsr()
    mst = minimum_spanning_tree(g)
    assert mst.nnz == len(res["edges"])
    assert np.isclose(mst.sum(), res["weight"] + len(res["edges"]), rtol=0, atol=1e-9)
    ncomp, labels = connected_components(g, directed=False)
    assert len(np.unique(res["root"])) == ncomp
    # same partition: the root is a function of the label and back
    assert len(set(zip(labels, res["root"]))) == ncomp
    # parent edges are the forest's edges, each root is its component's max z
    assert parent_edges(res["parent"]) == {tuple(e) for e in res["edges"].tolist()}
    for r in np.unique(res["root"]):
        members = np.nonzero(res["root"] == r)[0]
        top = members[np.lexsort((members, -p[members, 2]))[0]]
        assert top == r and res["parent"][r] == -1
    assert (np.abs(res["normals"]) == np.abs(n)).all()


def test_sphere_outward():
    p = _sphere(3000)
    idx = knn_rows(p, 20)
    n, _ = pca_normals(p, idx)
    assert (np.sum(n * p, 1) < 0).any()        # the canonical signs alone are not consistent
    res = orient(p, n, idx)
    assert (np.sum(res["normals"] * p, 1) > 0).all()
    assert len(np.unique(res["root"])) == 1
