"""The block-row algebra of kb200_append_data (DESIGN.md §5g) in numpy: with n0 = n rounded down to the 64-row tile,
rows [n0, n + m) are the new block row (the partial old tile row is factored again with the new rows), and

    L21 = C21 W11^T,  S = C22 - L21 L21^T,  L22 = chol(S),  W22 = L22^-1,  W21 = -W22 (L21 W11)

reproduce cholesky / inv of the full matrix, one append at a time, across the 64- and 256-row boundaries and along a
chain of appends that each start from the previous result."""
import numpy as np
import pytest

TILE = 64


def covariance(rng, n):
    P = rng.uniform(0.0, 1000.0, size=(n, 2))
    d = np.sqrt(((P[:, None, :] - P[None, :, :]) ** 2).sum(-1))
    return np.exp(-3.0 * d / 300.0) + 0.05 * np.eye(n), P


def extend(C, L, W, n):
    """The factor L and W = L^-1 of C[:n, :n] -> those of all of C, by the block-row formulas."""
    N = C.shape[0]
    n0 = n // TILE * TILE
    L11, W11 = L[:n0, :n0], W[:n0, :n0]
    C21, C22 = C[n0:, :n0], C[n0:, n0:]
    L21 = C21 @ W11.T
    L22 = np.linalg.cholesky(C22 - L21 @ L21.T)
    W22 = np.linalg.inv(L22)
    W22 = np.tril(W22)
    W21 = -W22 @ (L21 @ W11)
    Ln, Wn = np.zeros((N, N)), np.zeros((N, N))
    Ln[:n0, :n0], Ln[n0:, :n0], Ln[n0:, n0:] = L11, L21, L22
    Wn[:n0, :n0], Wn[n0:, :n0], Wn[n0:, n0:] = W11, W21, W22
    return Ln, Wn


def check(C, L, W, tol=1e-12):
    Lr = np.linalg.cholesky(C)
    Wr = np.linalg.inv(Lr)
    assert np.abs(L - Lr).max() <= tol * np.abs(Lr).max()
    assert np.abs(W - Wr).max() <= tol * np.abs(Wr).max() * 10
    assert np.abs(W @ L - np.eye(C.shape[0])).max() <= 1e-10


@pytest.mark.parametrize("n,m", [(1, 1), (1, 300), (63, 1), (63, 2), (64, 1), (64, 64), (65, 63), (127, 130),
                                 (255, 1), (256, 1), (256, 255), (257, 65), (300, 300), (511, 2), (600, 1),
                                 (600, 64), (512, 100)])
def test_one_append_reproduces_the_full_factor(n, m):
    rng = np.random.default_rng(n * 1000 + m)
    C, _ = covariance(rng, n + m)
    L0 = np.linalg.cholesky(C[:n, :n])
    L, W = extend(C, L0, np.linalg.inv(L0), n)
    check(C, L, W)


def test_chain_of_ten_appends():
    rng = np.random.default_rng(7)
    sizes = [50, 1, 13, 64, 65, 2, 100, 37, 63, 1, 120]
    C, _ = covariance(rng, sum(sizes))
    n = sizes[0]
    L = np.linalg.cholesky(C[:n, :n])
    W = np.linalg.inv(L)
    for m in sizes[1:]:
        L, W = extend(C[:n + m, :n + m], L, W, n)
        n += m
        check(C[:n, :n], L, W)
