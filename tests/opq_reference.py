"""Float64 reference of optimised-PQ indexes (`opq=1`), on top of tests/ivf_reference.py, pq4_reference.py and
pq_lut_reference.py.

An opq=1 index stores R [d][d] fp32 (row-major, y = x.R) and keeps its inverted-file side in the rotated space: the stored
centroids are C.R, the codebooks, codes and norm terms those of x.R, while the fp32 rows stay as given.  The first stage
probes and scans with the prepared query rotated; the exact second stage re-ranks from the unrotated rows with the prepared
query.

`read_index` decodes a B2IX v5 file: the v2 layout (reserved0 = 0) or the v3 one (4-bit codes, reserved0 = 4), followed by
R.  It strips R, patches the version and hands the rest to the existing readers.  `rotate_f32` reproduces the library's
rotation (one fmaf chain per element over the columns of x in order), so the reference's rotated query carries the same
fp32 value, and so the same bf16 rounding, as the device's.  `rotated` gives the stored index with its rows replaced by
their rotations, on which the existing list, code and key checks work unchanged.  numpy only: nothing here imports the
library."""
import os
import tempfile

import numpy as np

from tests import ivf_reference as R
from tests import pq4_reference as P
from tests import pq_lut_reference as L

VERSION = 5


def split_v5(raw):
    """v5 bytes -> (bytes of the v2 / v3 file without R, R float32 [d][d])."""
    h = np.frombuffer(raw, R.HEADER, count=1)[0]
    assert h["magic"] == b"B2IX" and h["version"] == VERSION, "not a B2IX v5 (OPQ) file"
    d = int(h["d"])
    tail = d * d * 4
    rot = np.frombuffer(raw[len(raw) - tail:], "<f4").reshape(d, d).astype(np.float32)
    body = bytearray(raw[:len(raw) - tail])
    hv = np.frombuffer(body, R.HEADER, count=1).copy()
    hv["version"] = 3 if int(h["reserved0"]) == 4 else 2
    body[:R.HEADER.itemsize] = hv.tobytes()
    return bytes(body), rot


def read_index(path):
    """(StoredIndex of the v2 / v3 part, R float32 [d][d], bits)."""
    body, rot = split_v5(open(path, "rb").read())
    bits = 4 if np.frombuffer(body, R.HEADER, count=1)[0]["version"] == 3 else 8
    fd, tmp = tempfile.mkstemp(suffix=".b2ix")
    try:
        with os.fdopen(fd, "wb") as f:
            f.write(body)
        s = P.read_index4(tmp) if bits == 4 else R.read_index(tmp)
    finally:
        os.unlink(tmp)
    return s, rot, bits


def orthonormal_error(rot):
    r = np.asarray(rot, np.float64)
    return float(np.abs(r.T @ r - np.eye(len(r))).max())


def rotate_f32(x, rot):
    """x [n][d] fp32 -> x.R in fp32, as the library computes it: acc = fmaf(x[i], R[i][j], acc) for i = 0 .. d - 1.  A float64
    product of two fp32 values is exact, and the float64 sum rounded to fp32 is fmaf's single rounding except in double-rounding
    corner cases (far below every tolerance the callers apply)."""
    x = np.asarray(x, np.float32)
    rot = np.asarray(rot, np.float32)
    acc = np.zeros((len(x), rot.shape[1]), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(rot.shape[0]):
            acc = (acc.astype(np.float64) + x[:, i:i + 1].astype(np.float64) * rot[i][None, :].astype(np.float64)).astype(np.float32)
    return acc


def rotated(s, rot):
    """A copy of the stored index with every row replaced by its rotation, x.R in float64 rounded to fp32 (within a few fp32
    units of the library's rows, far below the 1e-5 tolerances of the list and code checks): the index as the list side sees
    it."""
    t = s.copy()
    with np.errstate(invalid="ignore", over="ignore"):
        t.rows = (s.rows.astype(np.float64) @ np.asarray(rot, np.float64)).astype(np.float32)
    return t


def check_build(s, rot, bits, ix, y):
    """Build invariants of a stored opq=1 index: the fp32 rows as given (cosine: unit length), and, on the rotated rows, every
    usable row in the list of its nearest stored (rotated) centroid and no unusable one, the codes the nearest codewords of the
    rotated residual and the norm terms from those codes (the existing checks, run on `rotated`)."""
    y = np.asarray(y, np.float32)
    ok = R.usable(y)
    x = s.rows.astype(np.float32)
    if s.metric == R.COSINE:
        np.testing.assert_allclose(x[ok], R.normalize_rows_f32(y[ok]), rtol=0, atol=1e-6)
    else:
        assert x.tobytes() == y.tobytes(), "the stored fp32 rows differ from the input"
    t = rotated(s, rot)
    yr = t.rows.copy()
    yr[~ok] = np.nan          # unusable as given stays unusable (the rotation of an overflowing row need not overflow)
    t.rows = yr
    if s.metric == R.COSINE:  # check_lists compares the cosine rows with normalize(y): hand it rows it leaves as they are
        t.metric = R.IP
        t.bias = [None] * len(t.bias)
    (P.check_build if bits == 4 else L.check_build if L.is_lut(s) else R.check_build)(t, ix, yr)
    return t


def prepare_rotated(queries, metric, rot):
    """The library's first-stage queries: prepared (cosine: unit length), then rotated."""
    return rotate_f32(R.prepare_queries(queries, metric), rot)


def reference_search(s, rot, bits, queries, k, nprobe, alive=None):
    """tests/ivf_reference.reference_search for an opq=1 index: the keys of the stored (rotated) payload for the prepared,
    rotated queries; checked with ivf_reference.compare."""
    Q = prepare_rotated(queries, s.metric, rot)
    keys = P.row_keys if bits == 4 else L.row_keys if L.is_lut(s) else R.row_keys
    ids, lst, _ = s.flat()
    key, dis, tol = keys(s, Q)
    probed, allowed, flagged = R.coarse_probe(s, Q, nprobe)
    r = R.Reference()
    r.metric, r.k, r.nq = s.metric, k, len(Q)
    r.ids_all, r.lst_all, r.key, r.dis, r.tol = ids, lst, key, dis, tol
    r.allowed, r.flagged = allowed, flagged
    r.pos_of = {int(i): p for p, i in enumerate(ids.tolist())}
    r.ids = np.full((r.nq, k), -1, np.int64)
    r.out_dis = np.full((r.nq, k), -R.FLT_MAX if s.metric == R.IP else R.FLT_MAX)
    r.cand = []
    alive_row = np.ones(len(ids), bool) if alive is None else np.asarray(alive, bool)[ids]
    for q in range(r.nq):
        cand = np.nonzero(np.isin(lst, probed[q]) & alive_row)[0]
        cand = cand[np.lexsort((ids[cand], key[q, cand]))]
        r.cand.append(cand)
        top = cand[:k]
        r.ids[q, :len(top)] = ids[top]
        r.out_dis[q, :len(top)] = dis[q, top]
    r.alive_row = alive_row
    return r
