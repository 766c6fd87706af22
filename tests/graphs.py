"""Deterministic graph families for the kernel tests: scipy CSR float64 Laplacians L~ = 2 L / lmax - I (L the
normalised Laplacian I - D^-1/2 A D^-1/2; symmetric, spectrum in [-1, 1]).  Each family targets one branch of the
tile-metadata builder / launcher of the tensor-core conv (cheb_umma.cu: build_umma_level_meta, build_tileset,
umma_conv_supported, launch_n) — FAMILIES maps a name to (builder, the branch it targets)."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def _edges_to_adj(V, edges):
    e = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    e = e[e[:, 0] != e[:, 1]]
    A = sp.coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(V, V)).tocsr()
    A = ((A + A.T) > 0).astype(np.float64)
    return sp.csr_matrix(A)


def rescaled_laplacian(A: sp.spmatrix) -> sp.csr_matrix:
    """L~ = 2 L / lmax - I of the normalised Laplacian; an isolated vertex gets L_ii = 1 (one uniform diagonal)."""
    A = sp.csr_matrix(A, dtype=np.float64)
    V = A.shape[0]
    d = np.asarray(A.sum(axis=1)).ravel()
    inv = np.where(d > 0, 1.0 / np.sqrt(np.maximum(d, 1e-300)), 0.0)
    L = sp.identity(V, format="csr") - sp.diags(inv) @ A @ sp.diags(inv)
    L = sp.csr_matrix((L + L.T) / 2)
    lmax = lambda_max(L)
    Lt = sp.csr_matrix(2.0 / lmax * L - sp.identity(V, format="csr"))
    Lt.eliminate_zeros()
    Lt.sort_indices()
    return Lt


def lambda_max(L) -> float:
    if L.shape[0] <= 512:
        return float(np.linalg.eigvalsh(L.toarray()).max())
    return float(spla.eigsh(L, k=1, which="LA", return_eigenvectors=False, tol=1e-12)[0])


def path_chords(V, chord=7):
    """Path 0-1-...-(V-1) plus chords i ~ i + chord: degree <= 4, no edge longer than `chord`."""
    i = np.arange(V)
    return [(a, a + 1) for a in i[:-1]] + [(a, a + chord) for a in i[: max(V - chord, 0)]]


def sized(V):
    return rescaled_laplacian(_edges_to_adj(V, path_chords(V)))


def band(V, bw):
    """Every pair within distance bw: 128 + 2 bw one-hop rows and 128 (2 bw + 1) CSR entries per interior tile."""
    e = [(a, a + d) for d in range(1, bw + 1) for a in range(V - d)]
    return rescaled_laplacian(_edges_to_adj(V, e))


def far_edges(V, n_far):
    """Path + chords of length 2, and rows 0..n_far-1 (tile 0) joined to rows V-1, V-2, ... (the last tile): with
    rows 128 and 129 (the chords out of the tile), tile 0 stages 130 + n_far rows."""
    e = path_chords(V, chord=2) + [(i, V - 1 - i) for i in range(n_far)]
    return rescaled_laplacian(_edges_to_adj(V, e))


def hub(V=1024, n_spokes=60, seed=0):
    """Path graph plus one vertex (row 5) joined to n_spokes vertices spread over the whole graph: tile 0 stages its
    spokes as 1-hop rows, every spoke's tile stages the hub; |L~|'s row sum at the hub is far above 1 (the basis
    grows by (2 r^2 + 1) there)."""
    rng = np.random.default_rng(seed)
    spokes = rng.choice(np.arange(130, V), size=n_spokes, replace=False)
    e = path_chords(V, chord=2) + [(5, int(s)) for s in spokes]
    return rescaled_laplacian(_edges_to_adj(V, e))


def empty_rows(V=1024, every=5):
    """Rows (and columns) with no entry at all, not even a diagonal: T1 = 0 and T2 = -x there."""
    L = sp.lil_matrix(sized(V))
    dead = np.arange(3, V, every)
    keep = np.ones(V)
    keep[dead] = 0
    D = sp.diags(keep)
    out = sp.csr_matrix(D @ sp.csr_matrix(L) @ D)
    out.eliminate_zeros()
    out.sort_indices()
    return out


def isolated(V=1024, n_real=512, two_diagonals=False):
    """n_real connected rows, then V - n_real isolated rows (only a diagonal, 0.25).  One shared diagonal: padding
    elision builds its tile families; two different diagonals (every other isolated row -0.5): it must not."""
    L = sp.lil_matrix(rescaled_laplacian(_edges_to_adj(n_real, path_chords(n_real))).toarray())
    L.resize((V, V))
    for v in range(n_real, V):
        L[v, v] = -0.5 if (two_diagonals and v % 2) else 0.25
    out = sp.csr_matrix(L)
    out.sort_indices()
    return out


def band_far(V, bw, n_far):
    """band(V, bw) plus rows 0..n_far-1 joined to rows V-1, V-2, ...: tile 0 stages its band halo and n_far far rows
    on top of a band's CSR, so a large staged-row count and a large metadata blob come together."""
    e = [(a, a + d) for d in range(1, bw + 1) for a in range(V - d)] + [(i, V - 1 - i) for i in range(n_far)]
    return rescaled_laplacian(_edges_to_adj(V, e))


def block_clique(V, e, blk=64):
    """Cliques of blk consecutive vertices (one per 64-row tile), each vertex also joined to the first e vertices of
    the next block: a 64-row tile stages few rows (its block, the next e, the previous block) but holds a CSR entry for
    nearly every (own row, staged row) pair, so its metadata blob is large for its halo."""
    edges = []
    for b0 in range(0, V, blk):
        own = np.arange(b0, min(V, b0 + blk))
        nxt = np.arange(b0 + blk, min(V, b0 + blk + e))
        for other in (own, nxt):
            a, b = np.meshgrid(own, other)
            edges.append(np.stack([a.ravel(), b.ravel()], axis=1))
    return rescaled_laplacian(_edges_to_adj(V, np.concatenate(edges)))


def two_cliques(a):
    """Two 64-vertex cliques (one per 64-row tile), the last a vertices of the first joined to the first a of the
    second: each tile stages 64 + a rows and holds 64 * 64 + a * a CSR entries."""
    edges = [(i, j) for b0 in (0, 64) for i in range(b0, b0 + 64) for j in range(i + 1, b0 + 64)]
    edges += [(i, j) for i in range(64 - a, 64) for j in range(64, 64 + a)]
    return rescaled_laplacian(_edges_to_adj(128, edges))


def dense(V=2048, degree=64, seed=0):
    """Random graph of degree ~64: every 128-row tile stages far more than 512 rows (own rows + 1-hop halo), beyond
    what the tile-metadata builder accepts."""
    rng = np.random.default_rng(seed)
    a = np.repeat(np.arange(V), degree // 2)
    b = rng.integers(0, V, size=a.size)
    return rescaled_laplacian(_edges_to_adj(V, np.stack([a, b], axis=1)))


def nonsymmetric(V=256, seed=0):
    """A sparse matrix with L~ != L~^T (max absolute row and column sums < 1, so its spectrum is inside the disc)."""
    rng = np.random.default_rng(seed)
    M = sp.random(V, V, density=8.0 / V, random_state=np.random.RandomState(seed), format="csr")
    M.data = rng.uniform(-1, 1, size=M.data.size)
    M = M + sp.identity(V) * 0.25
    s = max(float(abs(M).sum(axis=1).max()), float(abs(M).sum(axis=0).max()))
    out = sp.csr_matrix(M / (1.01 * s))
    out.sort_indices()
    return out


# name -> (builder, branch)
FAMILIES = {
    **{f"V{V}": ((lambda V=V: sized(V)), "ragged last tile / V < 128 / TMA (V % 128 == 0) vs cp.async rows")
       for V in (1, 64, 127, 128, 129, 1088, 2048)},
    # band widths around the shared-memory limits (227 KB): 8, 12, 14: two X stages; 16: the conv drops to one;
    # 20: the conv still fits with one, the weight-gradient kernel no longer fits (SIMT dW)
    **{f"band{bw}": ((lambda bw=bw: band(1024, bw)), "X stages 2 -> 1 and the shared-memory cut-off to SIMT")
       for bw in (8, 12, 14, 16, 20)},
    # bands sized for the 64-row tiles of the 128- and 256-wide convs: 18, a ring of 3 slots in the 64 x 128
    # configuration; 21, the 64 x 256 mode with one T1 stage (tests/test_gpu_persistent_tiles_fp64.py)
    **{f"band{bw}": ((lambda bw=bw: band(1024, bw)), "64-row tiles: ring of 3 / one T1 stage") for bw in (18, 21)},
    "farband20": ((lambda: band_far(512, 20, 80)), "single-pass fp16, 128 x 64: one X stage"),
    **{f"clique{e}": ((lambda e=e: block_clique(512, e)), "64-row tiles with large blobs for their halo")
       for e in (12, 14)},
    # a = 49: the largest blobs for 113 staged rows that still fit a ring of 3 with one T1 stage; the 128-column plain
    # GEMM (the backward's dT GEMMs) then needs one X stage too
    "twoclique49": ((lambda: two_cliques(49)), "64-row tiles: the plain GEMM's ring of 3 with one X stage"),
    "h1_256": (lambda: far_edges(1024, 126), "max_h1 = 256: still tensor cores"),
    "h1_257": (lambda: far_edges(1024, 127), "max_h1 = 257: the 256-staged-row cut-off to SIMT"),
    "far": (lambda: far_edges(1088, 64), "halos that cross the whole graph (tile 0 <-> last, ragged) tile"),
    "hub": (hub, "one tile with a halo spread over the whole graph, |L~| row sum >> 1"),
    "empty_rows": (empty_rows, "rows with no entries"),
    "iso_uniform": (isolated, "isolated rows with one diagonal: elision tile families built"),
    "iso_two_diag": ((lambda: isolated(two_diagonals=True)), "isolated rows with two diagonals: no elision"),
    "dense": (dense, "tile metadata beyond the builder's caps: the level runs on SIMT"),
    "nonsymmetric": (nonsymmetric, "L~ != L~^T"),
}

_cache = {}


def get(name: str) -> sp.csr_matrix:
    if name not in _cache:
        _cache[name] = FAMILIES[name][0]()
    return _cache[name]


def torch_coo_with_duplicates(L):
    """The same matrix as a torch sparse COO tensor whose every entry is stored twice (v/2 + v/2, exact)."""
    import torch

    c = sp.coo_matrix(L)
    r = np.concatenate([c.row, c.row])
    k = np.concatenate([c.col, c.col])
    v = np.concatenate([c.data / 2, c.data / 2])
    order = np.random.default_rng(0).permutation(r.size)
    return torch.sparse_coo_tensor(np.stack([r[order], k[order]]), v[order], size=L.shape)
