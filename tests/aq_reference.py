"""Float64 reference of anisotropic product quantisation (`aq_threshold=T`, csrc/ivf_aq.cu), restated from the ScaNN paper
(Guo et al., ICML 2020) and the header comment of ivf_aq.cu.

  x        a row as indexed (unit length under cosine); c_l its list centroid; e_j its codeword in sub-space j
  x^       c_l + sum_j e_j;  r = x - x^;  a_j = x_j - c_l,j (the residual the codewords quantise)
  loss     l(x, x^) = ||r||^2 + w <r, x>^2,  w = (eta - 1) / ||x||^2  (w = 0 when ||x|| = 0)
  eta      (d - 1) T^2 / (1 - T^2): ScaNN's parallel-cost multiplier of a unit-norm row; eta = 1 when T^2 = 1 / d (plain PQ)

encode: start from the nearest codewords, then up to SWEEPS sweeps over j = 0 .. M - 1, stopping after a sweep that changed
no code.  With s = <r, x> - <r_j, x_j>, candidate e of sub-space j costs ||a_j - e||^2 + w (s + <a_j - e, x_j>)^2 up to a
constant; the code moves to the cheapest candidate (smallest index among equals) only when that is strictly cheaper.

train: from the k-means codebooks, ITERS iterations of: encode the sample; for j = 0 .. M - 1 solve, for every codeword e of
sub-space j with members S,
    (|S| I + sum_S w_i x_ij x_ij^T) e = sum_S [a_ij + w_i (<a_ij, x_ij> + s_ij) x_ij],   s_ij = p_i - <r_ij, x_ij>,  p_i = <r_i, x_i>
(a codeword without members keeps its value), then refresh every p_i.  The trajectory is the sample's mean loss after
encoding with the k-means codebooks, then after each iteration's update; the codebooks are rounded to fp32 after each solve,
as the device stores them.

The device decides in fp32 (u = 2^-24).  `encode` reports, per row, whether some decision of its path was within tol x u x
the scale of its terms of its runner-up: such a row is *ambiguous* and its device codes may differ.  Scales:
  nearest codeword:   sum over the two of (dsub + 2) (q_e + ||a_j|| sqrt(q_e)), q_e = ||a_j - e||^2: the fmaf sum of q_e
                      from a_j rounded to fp32;
  coordinate descent: sum over the two of (dsub + 2) (q_e + ||a_j|| sqrt(q_e)) + |w| (2 |pe_e| (dsub + 1) sqrt(q_e) ||x_j||
                      + 2 pe_e^2) + |l_e|, pe_e = s + dd_e, dd_e = <a_j - e, x_j> (their fp32 sums, the square, the fmaf),
                      plus 2 |w| (M + dsub) sum_k |<r_k, x_k>| |dd_1 - dd_2|: s, summed in fp32 from the per-sub-space
                      terms, is common to both candidates, so its error moves their difference only through dd_1 - dd_2.

numpy only: nothing here imports the library."""
import numpy as np

SWEEPS, ITERS = 4, 5     # kAqSweeps, kAqIters of csrc/ivf_aq.cu
MAX_DSUB = 64            # kAqMaxDsub
U = 2.0 ** -24
TOL_U = 16               # a decision is ambiguous when its margin is below TOL_U x u x the scale of its terms


def eta_of(d, t):
    return (d - 1) * t * t / (1.0 - t * t)


def weights(X, eta):
    xx = (X * X).sum(1)
    return np.where(xx > 0, (eta - 1.0) / np.where(xx > 0, xx, 1.0), 0.0)


def residual(X, C, lists, cb, codes):
    """r = x - c_l - sum_j e_j, float64 [n][d]."""
    m, _, dsub = cb.shape
    rec = np.concatenate([cb[j][codes[:, j]] for j in range(m)], axis=1)
    return X - C[lists] - rec


def row_loss(X, C, lists, cb, codes, eta):
    X, C, cb = (np.asarray(a, np.float64) for a in (X, C, cb))
    r = residual(X, C, lists, cb, codes)
    p = (r * X).sum(1)
    return (r * r).sum(1) + weights(X, eta) * p * p


def mean_loss(X, C, lists, cb, codes, eta):
    return float(row_loss(X, C, lists, cb, codes, eta).mean())


def nearest(X, C, lists, cb, tol=TOL_U):
    """Nearest codeword of every sub-vector of a = x - c_l (smallest index among equals), and which rows had a near tie."""
    X, C, cb = (np.asarray(a, np.float64) for a in (X, C, cb))
    m, ncw, dsub = cb.shape
    A = X - C[lists]
    codes = np.zeros((len(X), m), np.int64)
    amb = np.zeros(len(X), bool)
    for j in range(m):
        a = A[:, j * dsub:(j + 1) * dsub]
        e = cb[j]
        dist = (a * a).sum(1)[:, None] - 2 * a @ e.T + (e * e).sum(1)[None, :]
        codes[:, j] = np.argmin(dist, axis=1)
        if ncw > 1:
            two = np.argpartition(dist, 1, axis=1)[:, :2]
            d2 = np.take_along_axis(dist, two, 1)
            na = np.sqrt((a * a).sum(1))[:, None]
            scale = ((dsub + 2) * (d2 + na * np.sqrt(np.maximum(d2, 0)))).sum(1)
            amb |= np.abs(d2[:, 1] - d2[:, 0]) <= tol * U * scale
    return codes, amb


def encode(X, C, lists, cb, eta, codes0=None, sweeps=SWEEPS, tol=TOL_U):
    """Anisotropic codes of rows X [n][d] (float64 arithmetic).  Returns (codes [n][m], ambiguous [n], sweeps run [n])."""
    X, C, cb = (np.asarray(a, np.float64) for a in (X, C, cb))
    m, ncw, dsub = cb.shape
    n = len(X)
    if codes0 is None:
        codes, amb = nearest(X, C, lists, cb, tol)
    else:
        codes, amb = np.array(codes0, np.int64), np.zeros(n, bool)
    A = X - C[lists]
    w = weights(X, eta)
    rows = np.arange(n)
    # <r_k, x_k> per sub-space
    pd = np.stack([((A[:, k * dsub:(k + 1) * dsub] - cb[k][codes[:, k]]) * X[:, k * dsub:(k + 1) * dsub]).sum(1) for k in range(m)], 1)
    active = np.ones(n, bool)
    ran = np.zeros(n, np.int64)
    for _ in range(sweeps):
        if not active.any():
            break
        ran += active
        changed = np.zeros(n, bool)
        for j in range(m):
            a, x, e = A[:, j * dsub:(j + 1) * dsub], X[:, j * dsub:(j + 1) * dsub], cb[j]
            s = pd.sum(1) - pd[:, j]
            q = (a * a).sum(1)[:, None] - 2 * a @ e.T + (e * e).sum(1)[None, :]
            dd = (a * x).sum(1)[:, None] - x @ e.T
            pe = s[:, None] + dd
            cost = q + w[:, None] * pe * pe
            best = np.argmin(cost, axis=1)
            cur = codes[:, j]
            move = active & (cost[rows, best] < cost[rows, cur])
            # margin of the decision: the best against the runner-up (which may be the current code)
            if ncw > 1:
                two = np.argpartition(cost, 1, axis=1)[:, :2]
                c2, q2, d2, p2 = (np.take_along_axis(v, two, 1) for v in (cost, q, dd, pe))
                na, nx = np.sqrt((a * a).sum(1))[:, None], np.sqrt((x * x).sum(1))[:, None]
                sq = np.sqrt(np.maximum(q2, 0))
                aw = np.abs(w)[:, None]
                per = (dsub + 2) * (q2 + na * sq) + aw * (2 * np.abs(p2) * (dsub + 1) * sq * nx + 2 * p2 * p2) + np.abs(c2)
                common = 2 * aw[:, 0] * (m + dsub) * np.abs(pd).sum(1) * np.abs(d2[:, 1] - d2[:, 0])
                amb |= active & (np.abs(c2[:, 1] - c2[:, 0]) <= tol * U * (per.sum(1) + common))
            codes[move, j] = best[move]
            pd[move, j] = dd[rows, best][move]
            changed |= move
        active &= changed
    return codes, amb, ran


def update_block(X, C, lists, cb, codes, eta, j, p):
    """One block update of sub-space j: the new codebook of j (float64 solve of the normal equations, every codeword with
    members) and the per-codeword systems (A, b) for checking.  p: <r_i, x_i> of every row with the current codebooks."""
    X, C, cb = (np.asarray(a, np.float64) for a in (X, C, cb))
    m, ncw, dsub = cb.shape
    w = weights(X, eta)
    a = (X - C[lists])[:, j * dsub:(j + 1) * dsub]
    x = X[:, j * dsub:(j + 1) * dsub]
    new = cb[j].copy()
    onehot = (codes[:, j][None, :] == np.arange(ncw)[:, None]).astype(np.float64)   # [ncw][n]: members in row order
    count = onehot.sum(1)
    rx = ((a - cb[j][codes[:, j]]) * x).sum(1)
    beta = w * ((a * x).sum(1) + (p - rx))
    Amat = count[:, None, None] * np.eye(dsub) + (onehot @ (w[:, None] * (x[:, :, None] * x[:, None, :]).reshape(len(x), -1))).reshape(ncw, dsub, dsub)
    b = onehot @ (a + beta[:, None] * x)
    has = np.nonzero(count > 0)[0]   # a codeword without members keeps its value
    if len(has):
        new[has] = np.linalg.solve(Amat[has], b[has][:, :, None])[:, :, 0]
    systems = {int(e): (Amat[e], b[e]) for e in has}
    return new, systems


def train(X, C, lists, cb0, eta, iters=ITERS, tol=TOL_U):
    """The training trajectory from the k-means codebooks cb0 [m][ncw][dsub].  Returns (codebooks fp32, mean losses
    [1 + iters], number of ambiguous sample rows over all encodings)."""
    X, C = np.asarray(X, np.float64), np.asarray(C, np.float64)
    cb = np.asarray(cb0, np.float32).copy()
    m = cb.shape[0]
    traj, n_amb = [], 0
    for it in range(iters):
        codes, amb, _ = encode(X, C, lists, cb, eta, tol=tol)
        n_amb += int(amb.sum())
        if it == 0:
            traj.append(mean_loss(X, C, lists, cb, codes, eta))
        cb64 = cb.astype(np.float64)
        p = (residual(X, C, lists, cb64, codes) * X).sum(1)
        for j in range(m):
            new, _ = update_block(X, C, lists, cb64, codes, eta, j, p)
            new = new.astype(np.float32).astype(np.float64)
            dsub = cb.shape[2]
            p += ((cb64[j][codes[:, j]] - new[codes[:, j]]) * X[:, j * dsub:(j + 1) * dsub]).sum(1)
            cb64[j] = new
        cb = cb64.astype(np.float32)
        traj.append(mean_loss(X, C, lists, cb, codes, eta))
    return cb, np.array(traj), n_amb


def brute_force(X, C, lists, cb, eta):
    """The loss-optimal codes over every combination of codewords (small M and codebooks only)."""
    X, C, cb = (np.asarray(a, np.float64) for a in (X, C, cb))
    m, ncw, _ = cb.shape
    combos = np.array(np.meshgrid(*[np.arange(ncw)] * m, indexing="ij")).reshape(m, -1).T
    best = np.zeros((len(X), m), np.int64)
    for i in range(len(X)):
        Xi = np.repeat(X[i:i + 1], len(combos), 0)
        li = np.repeat(lists[i:i + 1], len(combos), 0)
        best[i] = combos[np.argmin(row_loss(Xi, C, li, cb, combos, eta))]
    return best
