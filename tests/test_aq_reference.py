"""The anisotropic-PQ reference (tests/aq_reference.py) against itself: the encoder never increases the loss and stops at a
fixed point, every block update solves its normal equations and does not increase the sample loss, eta = 1 is plain PQ,
and on small codebooks the encoder is compared with a search over every code combination.  CPU only."""
import numpy as np
import pytest

from tests import aq_reference as A


def _problem(seed, n=300, d=16, m=4, ncw=16, nlist=3, unit=True):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)) + 0.5
    if unit:
        X /= np.linalg.norm(X, axis=1, keepdims=True)
    lists = rng.integers(0, nlist, n)
    C = np.stack([X[lists == l].mean(0) if (lists == l).any() else np.zeros(d) for l in range(nlist)])
    dsub = d // m
    res = X - C[lists]
    cb = np.stack([res[rng.choice(n, ncw, replace=False), j * dsub:(j + 1) * dsub] for j in range(m)])
    return X, C, lists, cb.astype(np.float32).astype(np.float64)


def test_eta():
    assert A.eta_of(768, 0.2) == pytest.approx(767 * 0.04 / 0.96)
    d = 64
    assert A.eta_of(d, np.sqrt(1.0 / d)) == pytest.approx(1.0)


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("t", [0.2, 0.5])
def test_encoder_never_increases_the_loss_and_is_a_fixed_point(seed, t):
    X, C, lists, cb = _problem(seed)
    eta = A.eta_of(X.shape[1], t)
    near, _ = A.nearest(X, C, lists, cb)
    codes, _, ran = A.encode(X, C, lists, cb, eta)
    l0, l1 = A.row_loss(X, C, lists, cb, near, eta), A.row_loss(X, C, lists, cb, codes, eta)
    assert (l1 <= l0 + 1e-12).all()
    assert (l1 < l0 - 1e-9).any(), "the anisotropic loss should move some code on this data"
    # rows that stopped before the sweep limit are fixed points of one more sweep
    again, _, _ = A.encode(X, C, lists, cb, eta, codes0=codes, sweeps=1)
    done = ran < A.SWEEPS
    assert done.any()
    assert (again[done] == codes[done]).all()
    # and one more sweep never increases anyone's loss
    assert (A.row_loss(X, C, lists, cb, again, eta) <= l1 + 1e-12).all()


@pytest.mark.parametrize("seed", range(2))
def test_block_updates_solve_their_normal_equations_and_do_not_increase_the_loss(seed):
    X, C, lists, cb = _problem(seed, n=400)
    eta = A.eta_of(X.shape[1], 0.3)
    codes, _, _ = A.encode(X, C, lists, cb, eta)
    cb = cb.copy()
    m, ncw, dsub = cb.shape
    before = A.mean_loss(X, C, lists, cb, codes, eta)
    for j in range(m):
        p = (A.residual(X, C, lists, cb, codes) * X).sum(1)
        new, systems = A.update_block(X, C, lists, cb, codes, eta, j, p)
        for e, (Amat, b) in systems.items():
            assert np.allclose(Amat @ new[e], b, rtol=1e-10, atol=1e-10)
            assert np.all(np.linalg.eigvalsh(Amat) > 0)
        # no member: the codeword keeps its value
        for e in set(range(ncw)) - set(systems):
            assert (new[e] == cb[j][e]).all()
        cb[j] = new
        after = A.mean_loss(X, C, lists, cb, codes, eta)
        assert after <= before + 1e-12
        before = after


def test_training_trajectory_never_increases_within_an_iteration_and_ends_below_nearest():
    X, C, lists, cb = _problem(7, n=600)
    eta = A.eta_of(X.shape[1], 0.2)
    near, _ = A.nearest(X, C, lists, cb)
    plain = A.mean_loss(X, C, lists, cb, near, eta)
    cbf, traj, _ = A.train(X, C, lists, cb, eta)
    assert len(traj) == 1 + A.ITERS
    assert traj[0] <= plain
    assert traj[-1] < plain
    assert cbf.dtype == np.float32


def test_eta_one_is_plain_pq():
    X, C, lists, cb = _problem(3)
    d = X.shape[1]
    eta = A.eta_of(d, np.sqrt(1.0 / d))
    near, _ = A.nearest(X, C, lists, cb)
    codes, _, _ = A.encode(X, C, lists, cb, eta)
    assert (codes == near).all()
    # the update is the member mean
    j = 1
    p = (A.residual(X, C, lists, cb, codes) * X).sum(1)
    new, systems = A.update_block(X, C, lists, cb, codes, 1.0, j, p)
    dsub = cb.shape[2]
    a = (X - C[lists])[:, j * dsub:(j + 1) * dsub]
    for e in systems:
        assert np.allclose(new[e], a[codes[:, j] == e].mean(0), rtol=1e-12, atol=1e-12)


def test_m1_equals_brute_force():
    X, C, lists, cb = _problem(4, n=60, d=4, m=1, ncw=16)
    eta = A.eta_of(4, 0.6)
    codes, _, _ = A.encode(X, C, lists, cb, eta)
    assert (codes == A.brute_force(X, C, lists, cb, eta)).all()


@pytest.mark.parametrize("m", [2, 3])
def test_m2_m3_lie_between_optimum_and_nearest(m):
    X, C, lists, cb = _problem(5 + m, n=40, d=2 * m, m=m, ncw=8)
    eta = A.eta_of(2 * m, 0.6)
    near, _ = A.nearest(X, C, lists, cb)
    codes, _, _ = A.encode(X, C, lists, cb, eta)
    opt = A.brute_force(X, C, lists, cb, eta)
    lo, mid, hi = (A.row_loss(X, C, lists, cb, c, eta) for c in (opt, codes, near))
    assert (lo <= mid + 1e-12).all() and (mid <= hi + 1e-12).all()
