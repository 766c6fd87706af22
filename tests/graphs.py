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


def padded(V, real, edges):
    """V rows whose connected rows are `real` (ascending) joined by `edges` (pairs of positions in `real`), every other
    row isolated: one uniform diagonal, so padding elision builds its index-list tile families (DevLevel::real_tiles
    packs the connected rows 128 and 64 to a tile, iso_tiles the isolated ones)."""
    real = np.asarray(real)
    e = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    L = rescaled_laplacian(_edges_to_adj(V, real[e]))
    # isolated rows at 0.25, not 2 / lmax - 1: that is 0 (no entry at all) where the connected rows are bipartite
    iso = np.ones(V, dtype=bool)
    iso[real] = False
    L = sp.csr_matrix(L + sp.diags(np.where(iso, 0.25 - L.diagonal(), 0.0)))
    L.eliminate_zeros()
    L.sort_indices()
    return L


def pair_rows(V, n_real):
    """n_real connected rows of a padded level of V rows, the isolated ones in sibling pairs (2p, 2p + 1) spread evenly
    (an odd count: the last connected row isolated too): every 128-row tile of consecutive rows holds about the level's
    share of isolated rows, so the consecutive tiles stay small where the connected rows packed 128 to a tile do not."""
    n_iso = V - n_real
    iso = np.zeros(V // 2, dtype=bool)
    iso[(np.arange(n_iso // 2) * (V // 2)) // max(n_iso // 2, 1)] = True
    real = np.flatnonzero(~np.repeat(iso, 2))
    return real[:-1] if n_iso % 2 else real


def real_path_far(V, n_far):
    """Half the rows isolated (pair_rows); the connected ones a path in row order, the first n_far joined to the last
    n_far: the first connected-row tile stages 128 own rows, the next one and n_far far ones (max_h1 = 129 + n_far)."""
    real = pair_rows(V, V // 2)
    n = len(real)
    e = [(i, i + 1) for i in range(n - 1)] + [(i, n - 1 - i) for i in range(n_far)]
    return padded(V, real, e)


def real_cliques(V, c):
    """Half the rows isolated (pair_rows); the connected ones in cliques of c consecutive ones and a path through all: a
    connected-row tile holds ~128 c CSR entries, a consecutive tile only its share of connected rows' (half as many)."""
    real = pair_rows(V, V // 2)
    n = len(real)
    e = [(i, i + 1) for i in range(n - 1)]
    for b0 in range(0, n, c):
        blk = np.arange(b0, min(n, b0 + c))
        a, b = np.meshgrid(blk, blk)
        e += list(zip(a.ravel(), b.ravel()))
    return padded(V, real, e)


def real_count(V, n_real):
    """n_real connected rows (pair_rows; a path with chords of 7), the others isolated: the last connected-row tile is
    ragged unless n_real is a multiple of its tile size."""
    real = pair_rows(V, n_real)
    return padded(V, real, path_chords(len(real)))


def elision_hierarchy(level0, joints=17):
    """A MeshNet Laplacian list around one padded level: level0 (V rows), a level of V / 2 rows whose row p is
    connected iff row 2p or 2p + 1 of level0 is (so both children of an isolated row are isolated: the eval forward's
    dedup classes exist), its connected rows a path with chords of 7, and a joint graph of `joints` rows (a path)."""
    V = level0.shape[0]
    L0 = sp.csr_matrix(level0)
    iso0 = (np.diff(L0.indptr) == 1) & (L0.indices[L0.indptr[:-1]] == np.arange(V))
    real1 = np.flatnonzero(~(iso0[0::2] & iso0[1::2]))
    level1 = padded(V // 2, real1, path_chords(len(real1)))
    return [level0, level1, sized(joints)]


# MeshNet channels around an elision hierarchy (levels V, V / 2, joint): the padded level runs 128 -> 256 (two
# 128-column slices), 256 -> 256 (the 64 x 256 mode), 256 -> 64 (128 x 64), 64 -> 128 and the 128 -> 64 -> 3 head
ELISION_PLAN = [(5, 32, 64), (64, 128), (128, 256, 256, 64, 128), (128, 64, 3)]

# name -> (builder, what the padded level's index-list tiles target): every level has >= 128 isolated rows with one
# diagonal (tests/test_gpu_elision_tiles_fp64.py builds a MeshNet around it with elision_hierarchy)
ELISION = {
    "el_h1_256": (lambda: real_path_far(1024, 127), "connected-row tiles stage 256 rows: the max_h1 limit"),
    "el_h1_257": (lambda: real_path_far(1024, 128), "257 staged rows: no families, the level runs on consecutive tiles"),
    "el_clique24": (lambda: real_cliques(1024, 24), "64-row connected-row blobs: the 64 x 128 ring of 6, one T1 stage"),
    "el_clique40": (lambda: real_cliques(1024, 40), "the 64 x 128 ring of 3, 64 x 256 and 128 x 64 with one T1 stage"),
    "el_clique48": (lambda: real_cliques(1024, 48), "128-row connected-row blobs that fit no ring: no families"),
    "el_ragged": (lambda: real_count(1024, 600), "600 connected rows: the last tile ragged at 128 and at 64 rows"),
    "el_real128": (lambda: real_count(512, 128), "exactly one 128-row connected-row tile"),
    "el_real129": (lambda: real_count(512, 129), "129 connected rows: a second tile of one row"),
    **{f"el_iso{n}": ((lambda n=n: real_count(640, 640 - n)), f"{n} isolated rows of 640: 5 n_iso vs 2 V")
       for n in (255, 256, 257)},
    "el_rows2w": (lambda: real_count(256, 128), "V = 256: B V vs 2 width for the 256-wide convs"),
}


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


def elision(name: str) -> sp.csr_matrix:
    if name not in _cache:
        _cache[name] = ELISION[name][0]()
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
