"""Exact reference of a stored binary inverted-file index (BINARYIVF, and the BINARYHNSW / BINARYMSTG names it serves) and of
its search.

`read_binary_index` decodes a B2IX v2 file written by `VectorIndex.save` (layout: `index_save_io` in csrc/ivf.cu).
`reference_search` answers a batch from the decoded index alone: the coarse probe over the stored centroid bytes, then every
kept row of the probed lists keyed by the metric, and the top k by (key, id).  Every binary key is an integer below 2^24
(Jaccard: one IEEE fp32 division of two such integers), so the library must return these bytes exactly: `compare` allows
no tolerance.  numpy only: nothing here imports the library, so the reference cannot share a bug with it."""
import numpy as np

from tests import ivf_reference as R
from tests import train_reference as T

HAMMING, JACCARD = 3, 4
PAGE = R.PAGE
FLT_MAX = np.float32(np.finfo(np.float32).max)
WORK_BYTES = 1 << 25   # bytes of the temporary of one popcount block (bounds the reference's memory)


def round_up(a, b):
    return -(-a // b) * b


def geometry(row_bytes):
    """(kb_w, row_pad, cent_pad) of rows of `row_bytes` bytes, as b200_index_create derives them: k-blocks of the row rounded
    up to 16 bytes, at most 128 (one 1024-bit wgmma k-step); rows padded to whole k-blocks; centroids padded to 16 bytes."""
    kb_w = min(128, round_up(row_bytes, 16))
    return kb_w, round_up(row_bytes, kb_w), T.cent_pad(row_bytes)


class BinaryIndex:
    """The decoded file.  Header fields as attributes; rows u8 [n][row_bytes] or None; centroids u8 [nlist][cent_pad];
    list_len int64 [nlist].  Per list l: ids[l] u32, pool[l] u8 [len][row_pad] (the k-block-major pages unpacked),
    popc[l] fp32 (row_bias: the stored popcount of each row)."""

    def __init__(self):
        self.ids, self.pool, self.popc = [], [], []

    def copy(self):
        c = BinaryIndex()
        c.__dict__.update(self.__dict__)
        c.centroids = self.centroids.copy()
        c.list_len = self.list_len.copy()
        c.ids = [a.copy() for a in self.ids]
        c.pool = [a.copy() for a in self.pool]
        c.popc = [a.copy() for a in self.popc]
        return c

    def truncate_list(self, l, rows):
        """Keep the first `rows` rows of list l (a perturbation for negative controls)."""
        self.ids[l], self.pool[l], self.popc[l] = self.ids[l][:rows], self.pool[l][:rows], self.popc[l][:rows]
        self.list_len[l] = rows

    def flat(self):
        """All stored rows, list after list: (ids int64, list of each row, row bytes u8 [N][row_pad])."""
        lens = [len(a) for a in self.ids]
        ids = np.concatenate(self.ids).astype(np.int64)
        return ids, np.repeat(np.arange(self.nlist), lens), np.concatenate(self.pool)

    def locate(self, row_id):
        """(list, position in the list) of a stored row id."""
        for l in range(self.nlist):
            at = np.nonzero(self.ids[l] == row_id)[0]
            if len(at):
                return l, int(at[0])
        raise KeyError(row_id)


def read_binary_index(path):
    raw = open(path, "rb").read()
    h = np.frombuffer(raw, R.HEADER, count=1)[0]
    assert h["magic"] == b"B2IX" and h["version"] == 2, "not a B2IX v2 file"
    s = BinaryIndex()
    for f in R.HEADER.names:
        setattr(s, f, h[f].item() if f != "magic" else h[f])
    assert s.use_ivf and s.d % 8 == 0 and s.metric in (HAMMING, JACCARD), "binary inverted-file index expected"
    s.row_bytes = s.d // 8
    s.kb_w, s.row_pad, s.cent_pad = geometry(s.row_bytes)
    nl, n, rp, kw = s.nlist, s.n, s.row_pad, s.kb_w
    off = R.HEADER.itemsize

    def take(dtype, count):
        nonlocal off
        a = np.frombuffer(raw, dtype, count=count, offset=off)
        off += a.nbytes
        return a

    s.rows = take("u1", n * s.row_bytes).reshape(n, s.row_bytes) if s.has_raw else None
    s.centroids = take("u1", nl * s.cent_pad).reshape(nl, s.cent_pad).copy()
    s.list_len = take("<u4", nl).astype(np.int64)
    for l in range(nl):
        ln = int(s.list_len[l])
        pool, ids, popc = [], [], []
        for _ in range(-(-ln // PAGE)):
            pool.append(take("u1", PAGE * rp).reshape(rp // kw, PAGE, kw).transpose(1, 0, 2).reshape(PAGE, rp))
            ids.append(take("<u4", PAGE))
            popc.append(take("<f4", PAGE))
        s.pool.append(np.concatenate(pool)[:ln].copy() if pool else np.zeros((0, rp), np.uint8))
        s.ids.append(np.concatenate(ids)[:ln].astype(np.uint32) if ids else np.zeros(0, np.uint32))
        s.popc.append(np.concatenate(popc)[:ln].astype(np.float32) if popc else np.zeros(0, np.float32))
    assert off == len(raw), f"{len(raw) - off} bytes left after the last page"
    assert sum(-(-int(v) // PAGE) for v in s.list_len) == s.pages_used, "pages_used differs from the list lengths"
    return s


def popcount_rows(b):
    """Set bits of every row of u8 [rows][w]."""
    return np.bitwise_count(np.asarray(b, np.uint8)).sum(1, dtype=np.int64)


def check_binary_build(s, y):
    """Asserts that the stored index holds exactly the rows y (u8 [n][row_bytes]), each once, in its nearest list."""
    y = np.ascontiguousarray(y, np.uint8)
    n, rb = y.shape
    assert s.n == n and s.row_bytes == rb
    ids, lst, pool = s.flat()
    assert np.array_equal(np.sort(ids), np.arange(n)), "the stored ids are not a permutation of 0..n-1"
    assert np.array_equal(pool[:, :rb], y[ids]), "a stored row differs from the row of its id"
    assert not pool[:, rb:].any(), "row padding bytes are not zero"
    assert not s.centroids[:, rb:].any(), "centroid padding bytes are not zero"
    popc = np.concatenate(s.popc)
    assert np.array_equal(popc, popcount_rows(pool).astype(np.float32)), "a stored popcount differs from its row's"
    cbits = np.unpackbits(s.centroids[:, :rb], axis=1)
    step = max(1, (1 << 22) // (8 * rb))   # rows per block: hamming_argmin widens the bits to fp32
    near = np.concatenate([T.hamming_argmin(np.unpackbits(pool[r0:r0 + step, :rb], axis=1), cbits)
                           for r0 in range(0, len(pool), step)])
    bad = np.nonzero(near != lst)[0]
    assert not len(bad), f"{len(bad)} rows not in their nearest list (first: id {ids[bad[0]]} in list {lst[bad[0]]}, nearest {near[bad[0]]})"


def _words(a):
    return np.ascontiguousarray(a, np.uint8).view("<u8")


def coarse_distances(s, queries):
    """Hamming distance int64 [nq][nlist] of every query, zero-padded to cent_pad bytes, to every stored centroid.  The probe
    ranks lists by this distance under BOTH metrics: the centroid table is a Hamming corpus (upload_coarse_bin)."""
    q = np.ascontiguousarray(queries, np.uint8)
    qc = np.zeros((len(q), s.cent_pad), np.uint8)
    qc[:, :s.row_bytes] = q
    qw, cw = _words(qc), _words(s.centroids)
    out = np.empty((len(q), s.nlist), np.int64)
    step = max(1, WORK_BYTES // max(1, s.nlist * cw.shape[1] * 8))
    for q0 in range(0, len(q), step):
        out[q0:q0 + step] = np.bitwise_count(qw[q0:q0 + step, None, :] ^ cw[None, :, :]).sum(2, dtype=np.int64)
    return out


def coarse_probe(s, queries, nprobe, ties="smaller"):
    """Lists each query probes, int64 [nq][min(nprobe, nlist)]: ascending (distance, list id), every list when
    nprobe >= nlist.  ties="larger" breaks equal distances toward the larger list id (a perturbation for negative controls)."""
    dist = coarse_distances(s, queries)
    nl = s.nlist
    npr = max(1, min(int(nprobe), nl))
    if npr >= nl:
        return np.tile(np.arange(nl), (len(dist), 1))
    lid = np.arange(nl) if ties == "smaller" else nl - 1 - np.arange(nl)
    return np.argsort(dist * nl + lid[None, :], axis=1, kind="stable")[:, :npr]


def coarse_ties(s, queries, nprobe):
    """Per query: the nprobe-th and (nprobe+1)-th nearest centroids are at equal distance (the probe's tie rule decides
    which list is scanned)."""
    dist = np.sort(coarse_distances(s, queries), axis=1)
    if nprobe >= s.nlist or nprobe < 1:
        return np.zeros(len(dist), bool)
    return dist[:, nprobe - 1] == dist[:, nprobe]


class Reference:
    """ids int64 [nq][k], dis fp32 [nq][k] (the answer); probed [nq][nprobe'] (the lists each query scans)."""

    def head(self, nq, k):
        """The answer of the first nq queries at a smaller k (a prefix of every row: the order is total)."""
        r = Reference()
        r.ids, r.dis, r.probed = self.ids[:nq, :k], self.dis[:nq, :k], self.probed[:nq]
        return r


def reference_search(s, queries, k, nprobe, alive=None, coarse="smaller", ties="smaller"):
    """The answer of s to u8 queries [nq][row_bytes] at (k, nprobe).  alive: LSB-first bitmap (u8) of the rows that may be
    returned, or None.  Keys: Hamming popc(q ^ y); Jaccard (or - and) / or as one fp32 division, 0 when or == 0.  The top k
    by (key, id); slots past the kept rows hold id -1 and FLT_MAX.  coarse / ties = "larger" break coarse-probe ties and final
    ties toward the larger id instead (perturbations for negative controls)."""
    q = np.ascontiguousarray(queries, np.uint8)
    nq = len(q)
    assert q.shape[1] == s.row_bytes
    qp = np.zeros((nq, s.row_pad), np.uint8)
    qp[:, :s.row_bytes] = q
    qw = _words(qp)
    popq = popcount_rows(q)
    ids_all, _, pool = s.flat()
    yw = _words(pool)
    popy = popcount_rows(pool)
    starts = np.concatenate([[0], np.cumsum([len(a) for a in s.ids])])
    keep = np.ones(len(ids_all), bool)
    if alive is not None:
        keep = np.unpackbits(np.asarray(alive, np.uint8), bitorder="little")[ids_all].astype(bool)
    r = Reference()
    r.probed = coarse_probe(s, q, nprobe, coarse)
    r.ids = np.full((nq, k), -1, np.int64)
    r.dis = np.full((nq, k), FLT_MAX, np.float32)
    step = max(1, WORK_BYTES // (yw.shape[1] * 8))
    for i in range(nq):
        rows = np.concatenate([np.arange(starts[l], starts[l + 1]) for l in r.probed[i]])
        rows = rows[keep[rows]]
        x_and = np.empty(len(rows), np.int64)
        for r0 in range(0, len(rows), step):
            blk = rows[r0:r0 + step]
            x_and[r0:r0 + step] = np.bitwise_count(yw[blk] & qw[i][None, :]).sum(1, dtype=np.int64)
        x_or = popq[i] + popy[rows] - x_and
        if s.metric == HAMMING:
            key = (x_or - x_and).astype(np.float32)
        else:
            with np.errstate(divide="ignore", invalid="ignore"):
                key = np.where(x_or == 0, np.float32(0), (x_or - x_and).astype(np.float32) / x_or.astype(np.float32))
            key = key.astype(np.float32)
        rid = ids_all[rows]
        # keys are >= 0, so their fp32 bits order like the keys: one int64 sort key (key bits, id)
        tie = rid if ties == "smaller" else (1 << 32) - 1 - rid
        order = (key.view(np.int32).astype(np.int64) << 32) | tie
        m = min(k, len(order))
        if m == 0:
            continue
        top = np.argpartition(order, m - 1)[:m] if m < len(order) else np.arange(len(order))
        top = top[np.argsort(order[top], kind="stable")]
        r.ids[i, :m] = rid[top]
        r.dis[i, :m] = key[top]
    return r


def compare(ref, dis, ids):
    """Problems of a library answer against the reference (empty list: it passes): ids and fp32 distance bits must be equal in
    every slot, tails included."""
    ids = np.asarray(ids)
    dis = np.ascontiguousarray(dis, np.float32)
    if ids.shape != ref.ids.shape or dis.shape != ref.dis.shape:
        return [f"shape {ids.shape} / {dis.shape}, reference {ref.ids.shape}"]
    bad = (ids != ref.ids) | (dis.view(np.uint32) != ref.dis.view(np.uint32))
    if not bad.any():
        return []
    q, j = (int(v) for v in np.argwhere(bad)[0])
    return [f"{int(bad.sum())} slots differ in {int(bad.any(1).sum())} queries; first: query {q} slot {j}: "
            f"id {int(ids[q, j])} distance {dis[q, j]!r}, reference id {int(ref.ids[q, j])} distance {ref.dis[q, j]!r}"]
