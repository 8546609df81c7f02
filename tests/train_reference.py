"""Reference of index training: the coarse k-means, the SQ8 ranges, the PQ codebooks and the binary k-majority, restated step
by step from kmeans_device, kmajority_device, train_device_locked and b200_index_build (csrc/ivf.cu).

Float k-means runs in float64.  The device sums a cluster's members with fp32 atomics in any order, so a centroid is known
only to within a bound: every centroid coordinate carries `delta`, with |device - reference| <= delta as long as every
assignment of the trajectory is decided by more than the rounding of the device and the uncertainty of the centroids.  A
trajectory where some row's assignment is not so decided is *ambiguous*: a test built on it proves nothing, so tests assert
that their data is unambiguous before they compare.  The binary k-majority is integer work and is reproduced exactly.

Tolerance of an assignment (the device's fp32 distance of a row x to a centroid c, and its centroid bound):
  fp32:     (d + 16) u (|x|^2 + |c|^2 + 2 sum|x||c|), u = 2^-24: the worst case of the tiled kernel's d-term fmaf sums, and
            of the 3xTF32 tensor-core search (split error ~ 8u per product) taken by large tables;
  centroid: 2 sum (|x| + |c|) delta + sum delta^2 >= the change of |x - c|^2 when c moves by at most delta per coordinate.
A row is ambiguous when the runner-up is within the sum of both centroids' tolerances.  Bitwise-equal centroids with
delta = 0 are duplicate seeds: the device resolves them to the smaller id, exactly.

numpy only: nothing here imports the library.  File readers are those of tests/ivf_reference.py (v2) and
tests/pq4_reference.py (v3), plus `read_binary_coarse` for binary indexes."""
import numpy as np

from tests import ivf_reference as R

U = 2.0 ** -24
C1E3 = float(np.float32(1e-3))   # the split nudge's constant, as the fp32 literal 1e-3f
ASSIGN_CHUNK = 8192              # rows per distance block (bounds the reference's memory)


# ---------------------------------------------------------------------------------------------------------------------------
# build decisions (b200_index_build, decide_ivf)
# ---------------------------------------------------------------------------------------------------------------------------
def default_nlist(n):
    """nlist when no ncentroids is given: clamp(floor(4 sqrt(n)), 1, 65536)."""
    return int(max(1, min(65536, int(4.0 * np.sqrt(float(max(n, 1)))))))


def use_ivf(total, n, nlist):
    """Whether an index of `total` rows trained on `n` rows is an inverted file (else FLAT)."""
    return total >= max(2000, 8 * nlist) and n >= nlist


def strided(n, k):
    """floor(i n / k) for i < k, computed in double as the device does: the seed rows and the build() sample."""
    return (np.arange(k, dtype=np.float64) * float(n) / float(k)).astype(np.int64)


def sample_rows(n, nlist):
    """Rows of an n-row build() that train the index: all of them when n <= max(256 nlist, 65536), else that many strided."""
    ns = min(n, max(256 * max(nlist, 1), 65536))
    return np.arange(n) if ns == n else strided(n, ns)


def build_sample(y, nlist):
    """The training rows of build(y) for an index with `nlist` lists (0: the default)."""
    n = len(y)
    nl = nlist if nlist > 0 else default_nlist(n)
    return y[sample_rows(n, nl)]


# ---------------------------------------------------------------------------------------------------------------------------
# float k-means
# ---------------------------------------------------------------------------------------------------------------------------
class Trajectory:
    """centroids float64 [nc][d] and delta [nc][d]; ambiguous + why (first few reasons); events: splits (pairs made),
    tied_splits (pairings where equal counts were broken by the smaller id), empties (empty clusters seen after updates,
    summed over iterations), empty_final (empty after the last update), last_change (the last iteration whose assignment
    differs from the one before, 0 if none), counts (weights per cluster of the last assignment)."""

    def __init__(self):
        self.ambiguous, self.why = False, []
        self.splits = self.tied_splits = self.empties = self.empty_final = self.last_change = 0

    def flag(self, msg):
        self.ambiguous = True
        if len(self.why) < 5:
            self.why.append(msg)


def assign_tol_rel(d):
    return (d + 16) * U


def assign(X, C, D, w_tol=None):
    """Nearest centroid of every row of X (float64) by L2, ties to the smaller id, and per row whether it is ambiguous (see
    the module docstring).  D: per-coordinate centroid bounds (zeros for exact centroids)."""
    n, d = X.shape
    nc = len(C)
    rel = assign_tol_rel(d) if w_tol is None else w_tol
    cc = (C * C).sum(1)
    aC = np.abs(C)
    unc_c = (aC * D).sum(1) * 2 + (D * D).sum(1)
    exact = ~D.any(1)
    same = np.unique(C, axis=0, return_inverse=True)[1].reshape(-1)   # equal centroids share a label
    best = np.empty(n, np.int64)
    amb = np.zeros(n, bool)
    for r0 in range(0, n, ASSIGN_CHUNK):
        x = X[r0:r0 + ASSIGN_CHUNK]
        ax = np.abs(x)
        xx = (x * x).sum(1)[:, None]
        dist = xx + cc[None, :] - 2.0 * (x @ C.T)
        b = np.argmin(dist, axis=1)
        rows = np.arange(len(x))
        tol = rel * (xx + cc[None, :] + 2.0 * (ax @ aC.T)) + 2.0 * (ax @ D.T) + unc_c[None, :]
        margin = dist - dist[rows, b][:, None]
        close = margin <= tol + tol[rows, b][:, None]
        close[rows, b] = False
        # duplicate seeds: bitwise-equal exact centroids are resolved to the smaller id, exactly
        close &= ~((same[None, :] == same[b][:, None]) & exact[None, :] & exact[b][:, None])
        best[r0:r0 + len(x)] = b
        amb[r0:r0 + len(x)] = close.any(1)
    return best, amb


def split_pairs(cnt):
    """(dst, src) pairs of the split rule for member counts cnt: the empty clusters in id order take the clusters sorted by
    count, largest first and equal counts by the smaller id, while those have at least 2 members.  Also returns how many
    pairs a count tie decided (their source ties with the cluster sorted before or after it)."""
    cnt = np.asarray(cnt)
    order = np.lexsort((np.arange(len(cnt)), -cnt))
    pairs, tied = [], 0
    for e, dst in enumerate(np.nonzero(cnt == 0)[0]):
        src = order[e]
        if cnt[src] < 2:
            break
        if (e + 1 < len(cnt) and cnt[order[e + 1]] == cnt[src]) or (e > 0 and cnt[order[e - 1]] == cnt[src]):
            tied += 1
        pairs.append((int(dst), int(src)))
    return pairs, tied


def kmeans(x, nc, iters, w=None, seeds=None, tol_rel=None):
    """kmeans_device on the fp32 rows x [n][d] (weights w: row i stands for w[i] identical rows; seeds: the initial rows,
    default floor(i n / nc)).  Returns a Trajectory."""
    x = np.asarray(x, np.float32)
    X = x.astype(np.float64)
    n, d = X.shape
    w = np.ones(n) if w is None else np.asarray(w, np.float64)
    seeds = strided(n, nc) if seeds is None else np.asarray(seeds, np.int64)
    C = X[seeds].copy()
    D = np.zeros_like(C)
    aX = np.abs(X)
    eps = np.where(np.arange(d) & 1, 1.0 / 1024, -1.0 / 1024)
    t = Trajectory()
    prev = None
    for it in range(iters):
        a, amb = assign(X, C, D, tol_rel)
        if amb.any():
            t.flag(f"iteration {it}: {int(amb.sum())} rows within tolerance of a second centroid (first: row {int(np.argmax(amb))})")
        if prev is not None and (a != prev).any():
            t.last_change = it
        prev = a
        cnt = np.bincount(a, weights=w, minlength=nc)
        S = np.empty((nc, d))
        A = np.empty((nc, d))
        for j in range(d):
            S[:, j] = np.bincount(a, weights=w * X[:, j], minlength=nc)
            A[:, j] = np.bincount(a, weights=w * aX[:, j], minlength=nc)
        nz = cnt > 0
        k = cnt[nz][:, None]
        mean = S[nz] / k
        C[nz] = mean
        # recursive fp32 summation of cnt terms (any order) + the rounding of the division
        D[nz] = ((k - 1) * U / (1 - (k - 1) * U)) * A[nz] / k + U * np.abs(mean)
        D[cnt == 1] = 0.0   # one member: 0 + x and x / 1 are exact
        empties = np.nonzero(~nz)[0]
        t.empties += len(empties)
        t.empty_final = len(empties)
        t.counts = cnt
        if it + 1 < iters and nc >= 2 and len(empties):
            pairs, tied = split_pairs(cnt)
            t.tied_splits += tied
            for dst, src in pairs:
                v, dv = C[src].copy(), D[src].copy()
                C[dst] = v * (1 + eps) + eps * C1E3
                C[src] = v * (1 - eps) - eps * C1E3
                D[dst] = dv * (1 + 1.0 / 1024) + U * (np.abs(v * (1 + eps)) + np.abs(C[dst]))
                D[src] = dv * (1 + 1.0 / 1024) + U * (np.abs(v * (1 - eps)) + np.abs(C[src]))
                t.splits += 1
    t.centroids, t.delta = C, D
    return t


def centroid_problems(got, t, what="centroid"):
    """Coordinates of the device's centroids `got` [nc][d] outside the reference's bound (empty list: they match)."""
    got = np.asarray(got, np.float64)
    err = np.abs(got - t.centroids)
    bad = err > t.delta
    if not bad.any():
        return []
    out = []
    for c, j in zip(*np.nonzero(bad)):
        if len(out) == 6:
            break
        out.append(f"{what} {c} coord {j}: device {got[c, j]!r}, reference {t.centroids[c, j]!r} (bound {t.delta[c, j]:.3g})")
    return [f"{int(bad.sum())} coordinates outside the bound"] + out


# ---------------------------------------------------------------------------------------------------------------------------
# SQ8 ranges and PQ codebooks (train_device_locked)
# ---------------------------------------------------------------------------------------------------------------------------
def train_rows(y, metric):
    """The rows the index trains on: unit length under cosine (the device's normalisation)."""
    y = np.ascontiguousarray(y, np.float32)
    return R.normalize_rows_f32(y) if metric == R.COSINE else y


def sq_ranges(x, fused_mid=False):
    """[4][d] fp32: lo, step, 1 / step, mid as the host computes them from the per-dimension min / max of the training rows.
    128 step is exact, so mid is the same with or without a fused multiply-add; fused_mid computes it fused anyway."""
    x = np.asarray(x, np.float32)
    lo, hi = x.min(0), x.max(0)
    with np.errstate(over="ignore"):
        step = np.where(hi > lo, (hi - lo) / np.float32(255), np.float32(1)).astype(np.float32)
    inv = (np.float32(1) / step).astype(np.float32)
    if fused_mid:
        mid = (lo.astype(np.float64) + 128.0 * step.astype(np.float64)).astype(np.float32)
    else:
        mid = (lo + np.float32(128) * step).astype(np.float32)
    return np.stack([lo, step, inv, mid])


def sq_problems(got, want_rows):
    """Differences of a stored SQ8 range table got [4][d] (lo, step, 1 / step, mid) from the reference of the rows, bit for
    bit (mid may also be the fused form)."""
    want = sq_ranges(want_rows)
    fused = sq_ranges(want_rows, fused_mid=True)
    bad = []
    for i, name in enumerate(("lo", "step", "1/step", "mid")):
        ok = got[i] == want[i]
        if i == 3:
            ok |= got[i] == fused[i]
        if not ok.all():
            j = int(np.argmin(ok))
            bad.append(f"{name}[{j}]: device {got[i][j]!r}, reference {want[i][j]!r}")
    return bad


def pq_sample(x, stride_rule="first"):
    """The PQ training sample: the first ns = min(n, 65536) rows of the view strided by max(1, n // ns).  stride_rule="even"
    takes rows floor(i n / ns) instead (a perturbation for negative controls)."""
    n = len(x)
    ns = min(n, 65536)
    if stride_rule == "even":
        return x[strided(n, ns)]
    return x[::max(1, n // ns)][:ns]


class PQTraining:
    """subs: one Trajectory per sub-quantiser; coarse_ambiguous: rows of the sample whose list is not decided; ambiguous:
    any of it."""


def pq_codebooks(x, centroids, m, bits, stride_rule="first"):
    """Codebooks of a PQ index trained on rows x (prepared: unit length under cosine) with the stored coarse centroids:
    the sample, its exact coarse assignment, its fp32 residuals, and per sub-quantiser k-means (256 or 16 codewords,
    8 iterations)."""
    x = np.asarray(x, np.float32)
    d = x.shape[1]
    dsub = d // m
    samp = pq_sample(x, stride_rule)
    C = np.asarray(centroids, np.float32)
    lst, amb = assign(samp.astype(np.float64), C.astype(np.float64), np.zeros((len(C), d)))
    res = (samp - C[lst]).astype(np.float32)   # residual_sub_kernel: one fp32 subtraction
    p = PQTraining()
    p.coarse_ambiguous = int(amb.sum())
    p.subs = [kmeans(res[:, j * dsub:(j + 1) * dsub], 16 if bits == 4 else 256, 8) for j in range(m)]
    p.ambiguous = p.coarse_ambiguous > 0 or any(s.ambiguous for s in p.subs)
    return p


def codebook_problems(codebook, p):
    out = []
    for j, s in enumerate(p.subs):
        out += centroid_problems(codebook[j], s, f"sub-quantiser {j} codeword")
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# binary k-majority (kmajority_device) and the binary index file
# ---------------------------------------------------------------------------------------------------------------------------
def cent_pad(row_bytes):
    return -(-row_bytes // 16) * 16


def hamming_argmin(bits, C):
    """Nearest centroid by Hamming distance, ties to the smaller id: bits [n][nbits], C [nc][nbits] as 0 / 1 (exact in fp32:
    every sum is below 2^24)."""
    a = bits.astype(np.float32)
    c = C.astype(np.float32)
    out = np.empty(len(a), np.int64)
    for r0 in range(0, len(a), ASSIGN_CHUNK):
        blk = a[r0:r0 + ASSIGN_CHUNK]
        ham = blk.sum(1)[:, None] + c.sum(1)[None, :] - 2 * (blk @ c.T)
        out[r0:r0 + len(blk)] = np.argmin(ham, axis=1)
    return out


class BinTrajectory:
    """centroids u8 [nc][cent_pad]; iterations (updates made), stopped_early, splits, ties (member-count ties on a bit of a
    non-empty cluster, summed over updates), empty_final."""


def kmajority(xbytes, nc, iters, tie_sets=False):
    """kmajority_device on binary rows [n][row_bytes] u8.  tie_sets=True sets a bit on an exact tie instead of keeping it (a
    perturbation for negative controls)."""
    xb = np.ascontiguousarray(xbytes, np.uint8)
    n, rb = xb.shape
    bits = np.unpackbits(xb, axis=1, bitorder="little")
    C = bits[strided(n, nc)].copy()
    t = BinTrajectory()
    t.iterations, t.stopped_early, t.splits, t.ties, t.empty_final = 0, False, 0, 0, 0
    prev = np.full(n, -1)
    for it in range(iters):
        a = hamming_argmin(bits, C)
        changed = int((a != prev).sum())
        prev = a
        if it > 0 and changed == 0:
            t.stopped_early = True
            break
        cnt = np.bincount(a, minlength=nc)
        ones = np.zeros((nc, bits.shape[1]), np.int64)
        srt = np.argsort(a, kind="stable")
        live = np.nonzero(cnt)[0]
        ones[live] = np.add.reduceat(bits[srt], np.concatenate([[0], np.cumsum(cnt)[:-1]])[live], axis=0, dtype=np.int64)
        twice, m = 2 * ones, cnt[:, None]
        tie = (twice == m) & (m > 0)
        t.ties += int(tie.sum())
        C = np.where(twice > m, 1, np.where(twice < m, 0, C)).astype(np.uint8)
        if tie_sets:
            C[tie] = 1
        t.iterations = it + 1
        t.empty_final = int((cnt == 0).sum())
        if it + 1 < iters and nc >= 2:
            for dst, src in split_pairs(cnt)[0]:
                C[dst] = bits[np.nonzero(a == src)[0][cnt[src] // 2]]   # the middle member, in row order
                t.splits += 1
    out = np.zeros((nc, cent_pad(rb)), np.uint8)
    out[:, :rb] = np.packbits(C, axis=1, bitorder="little")
    t.centroids = out
    t.assign_bits = C
    return t


def bin_list_lengths(xbytes, t):
    """List lengths of rows added to an index with the trajectory's final centroids (exact Hamming assignment)."""
    bits = np.unpackbits(np.ascontiguousarray(xbytes, np.uint8), axis=1, bitorder="little")
    return np.bincount(hamming_argmin(bits, t.assign_bits), minlength=len(t.centroids))


def read_binary_coarse(path):
    """(decoded index, centroid bytes u8 [nlist][cent_pad], list lengths int64 [nlist]) of a binary inverted-file index file,
    decoded whole by tests/binary_ivf_reference.read_binary_index."""
    from tests import binary_ivf_reference as B   # that module builds on this one
    s = B.read_binary_index(path)
    return s, s.centroids, s.list_len
