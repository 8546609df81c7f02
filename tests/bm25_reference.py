"""Float64 reference of BM25 text search and hybrid fusion, written from the published definitions (numpy only).

It shares nothing with the library or the C oracle: documents come in as per-field lists of TOKENS (the test generator
knows them by construction, so no tokenizer is restated), the field-norm code is tantivy's literal table
(``fieldnorm/code.rs``), and scores are summed in float64.  The only fp32 quantities are the ones tantivy itself defines
in fp32: the average field length, the 256-entry norm cache and the idf argument ``1 + (N - n + 0.5) / (n + 0.5)``
(for very common terms ``1 + x`` drops most of ``x`` in fp32, so a float64 idf would be off by up to 10 %).

``compare`` / ``compare_fusion`` return a list of problems (empty = accepted) for a result list the library returned.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
K1, B = 1.2, 0.75
MAX_TERMS = 64

# tantivy fieldnorm/code.rs FIELD_NORMS_TABLE: ids 0..39 are exact lengths, then 8 ids per doubling of the step
FIELDNORM_TABLE = np.array([
    0, 1, 2, 3, 4, 5, 6, 7,
    8, 9, 10, 11, 12, 13, 14, 15,
    16, 17, 18, 19, 20, 21, 22, 23,
    24, 25, 26, 27, 28, 29, 30, 31,
    32, 33, 34, 35, 36, 37, 38, 39,
    40, 42, 44, 46, 48, 50, 52, 54,
    56, 60, 64, 68, 72, 76, 80, 84,
    88, 96, 104, 112, 120, 128, 136, 144,
    152, 168, 184, 200, 216, 232, 248, 264,
    280, 312, 344, 376, 408, 440, 472, 504,
    536, 600, 664, 728, 792, 856, 920, 984,
    1048, 1176, 1304, 1432, 1560, 1688, 1816, 1944,
    2072, 2328, 2584, 2840, 3096, 3352, 3608, 3864,
    4120, 4632, 5144, 5656, 6168, 6680, 7192, 7704,
    8216, 9240, 10264, 11288, 12312, 13336, 14360, 15384,
    16408, 18456, 20504, 22552, 24600, 26648, 28696, 30744,
    32792, 36888, 40984, 45080, 49176, 53272, 57368, 61464,
    65560, 73752, 81944, 90136, 98328, 106520, 114712, 122904,
    131096, 147480, 163864, 180248, 196632, 213016, 229400, 245784,
    262168, 294936, 327704, 360472, 393240, 426008, 458776, 491544,
    524312, 589848, 655384, 720920, 786456, 851992, 917528, 983064,
    1048600, 1179672, 1310744, 1441816, 1572888, 1703960, 1835032, 1966104,
    2097176, 2359320, 2621464, 2883608, 3145752, 3407896, 3670040, 3932184,
    4194328, 4718616, 5242904, 5767192, 6291480, 6815768, 7340056, 7864344,
    8388632, 9437208, 10485784, 11534360, 12582936, 13631512, 14680088, 15728664,
    16777240, 18874392, 20971544, 23068696, 25165848, 27263000, 29360152, 31457304,
    33554456, 37748760, 41943064, 46137368, 50331672, 54525976, 58720280, 62914584,
    67108888, 75497496, 83886104, 92274712, 100663320, 109051928, 117440536, 125829144,
    134217752, 150994968, 167772184, 184549400, 201326616, 218103832, 234881048, 251658264,
    268435480, 301989912, 335544344, 369098776, 402653208, 436207640, 469762072, 503316504,
    536870936, 603979800, 671088664, 738197528, 805306392, 872415256, 939524120, 1006632984,
    1073741848, 1207959576, 1342177304, 1476395032, 1610612760, 1744830488, 1879048216, 2013265944,
], np.int64)


def fieldnorm_code(length):
    """The largest id whose table entry is <= the length."""
    return np.searchsorted(FIELDNORM_TABLE, np.asarray(length, np.int64), side="right") - 1


def distinct_terms(tokens):
    """The first 64 distinct terms of a query, in order."""
    out = []
    for t in tokens:
        if t not in out:
            out.append(t)
            if len(out) == MAX_TERMS:
                break
    return out


class RefResult:
    """Every matching live document of one query: row id, doc ordinal, float64 score and its tolerance."""

    def __init__(self, rows, ords, score, tol):
        self.rows, self.ords, self.score, self.tol = rows, ords, score, tol
        self.pos = {int(r): i for i, r in enumerate(rows.tolist())}

    def topk(self, k):
        """The expected list: fp32 scores descending, bit-equal scores by ascending doc ordinal."""
        s32 = self.score.astype(F32)
        order = np.lexsort((self.ords, -s32.astype(np.float64)))[:k]
        return self.rows[order], s32[order]


class BM25Reference:
    """fields[f] = (offsets[n_docs + 1], token ids) into vocab (lowercase terms); row_ids[n_docs]."""

    def __init__(self, vocab, fields, row_ids, quantise_lengths=True):
        self.vocab = list(vocab)
        self.term_id = {t: i for i, t in enumerate(self.vocab)}
        self.row_ids = np.asarray(row_ids, np.int64)
        self.n_docs = len(self.row_ids)
        self.n_fields = len(fields)
        self.quantise_lengths = quantise_lengths   # False: the raw length instead of its code (a negative control)
        nv = len(self.vocab)
        self.lens, self.total_tokens, self.post = [], [], []
        for offsets, ids in fields:
            offsets = np.asarray(offsets, np.int64)
            ids = np.asarray(ids, np.int64)
            lens = np.diff(offsets)
            doc = np.repeat(np.arange(self.n_docs, dtype=np.int64), lens)
            keys, tf = np.unique(ids * max(self.n_docs, 1) + doc, return_counts=True)
            term, pdoc = keys // max(self.n_docs, 1), keys % max(self.n_docs, 1)
            ptr = np.searchsorted(term, np.arange(nv + 1))
            self.lens.append(lens)
            self.total_tokens.append(int(lens.sum()))
            self.post.append((ptr, pdoc, tf.astype(np.float64)))

    @classmethod
    def from_tokens(cls, docs, row_ids, **kw):
        """docs[d][f] = list of tokens (str)."""
        n_fields = len(docs[0]) if docs else 1
        vocab, tid = [], {}
        fields = []
        for f in range(n_fields):
            offsets, ids = [0], []
            for d in docs:
                for t in d[f]:
                    if t not in tid:
                        tid[t] = len(vocab)
                        vocab.append(t)
                    ids.append(tid[t])
                offsets.append(len(ids))
            fields.append((offsets, ids))
        return cls(vocab, fields, row_ids, **kw)

    def doc_freq(self, term, field):
        t = self.term_id.get(term)
        if t is None:
            return 0
        ptr = self.post[field][0]
        return int(ptr[t + 1] - ptr[t])

    def stats(self):
        """This corpus' statistics in the form search(stats=...) takes."""
        df = {}
        for f in range(self.n_fields):
            ptr = self.post[f][0]
            for t in np.nonzero(np.diff(ptr))[0]:
                df[(f, self.vocab[t])] = int(ptr[t + 1] - ptr[t])
        return dict(total_docs=self.n_docs, total_tokens={f: self.total_tokens[f] for f in range(self.n_fields)}, doc_freq=df)

    def clause_contributions(self, field, term, stats=None):
        """(doc ordinals, float64 contributions) of one (field, term) clause."""
        t = self.term_id.get(term)
        ptr, pdoc, ptf = self.post[field]
        if t is None or ptr[t] == ptr[t + 1]:
            return np.zeros(0, np.int64), np.zeros(0)
        docs, tf = pdoc[ptr[t]:ptr[t + 1]], ptf[ptr[t]:ptr[t + 1]]
        N = int(stats["total_docs"]) if stats else self.n_docs
        T = int(stats["total_tokens"][field]) if stats else self.total_tokens[field]
        n = int(stats["doc_freq"].get((field, term), 0)) if stats else len(docs)
        avgdl = F32(T) / F32(N)
        dl = self.lens[field][docs]
        fn = FIELDNORM_TABLE[fieldnorm_code(dl)] if self.quantise_lengths else dl
        norm = (F32(K1) * ((F32(1) - F32(B)) + (F32(B) * fn.astype(F32)) / avgdl)).astype(np.float64)
        arg = F32(1) + (F32(N - n) + F32(0.5)) / (F32(n) + F32(0.5))
        idf = np.log(np.float64(arg))
        return docs, idf * (1.0 + K1) * tf / (tf + norm)

    def search(self, tokens, fields=(0,), alive=None, operator_or=True, stats=None):
        """tokens: the query's tokens (lowercase); alive: bool array over row ids or None."""
        terms = distinct_terms(tokens)
        nd = self.n_docs
        score, mag, m = np.zeros(nd), np.zeros(nd), np.zeros(nd)
        n_terms_hit = np.zeros(nd, np.int64)
        for term in terms:
            hit = np.zeros(nd, bool)
            for f in fields:
                docs, c = self.clause_contributions(f, term, stats)
                score += np.bincount(docs, c, nd)
                mag += np.bincount(docs, np.abs(c), nd)
                m += np.bincount(docs, None, nd)
                hit[docs] = True
            n_terms_hit += hit
        match = n_terms_hit > 0 if operator_or else (n_terms_hit == len(terms)) & (len(terms) > 0)
        if alive is not None:
            alive = np.asarray(alive, bool)
            match &= alive[self.row_ids]
        ords = np.nonzero(match)[0]
        return RefResult(self.row_ids[ords], ords, score[ords], 1e-6 * (m[ords] + 1) * mag[ords])


def _kth_checks(problems, ref_score, ref_tol, returned_idx, want, label):
    """Nothing clearly above the k-th reference score missing, nothing clearly below it returned."""
    if not want:
        return
    order = np.argsort(-ref_score, kind="stable")
    sk, tk = ref_score[order[want - 1]], ref_tol[order[want - 1]]
    got = np.zeros(len(ref_score), bool)
    got[returned_idx] = True
    missing = np.nonzero((ref_score - ref_tol > sk + tk) & ~got)[0]
    for i in missing[:5]:
        problems.append(f"{label(i)} (reference {ref_score[i]!r}) is above the k-th score {sk!r} but missing")
    for i in returned_idx:
        if ref_score[i] + ref_tol[i] < sk - tk:
            problems.append(f"{label(i)} (reference {ref_score[i]!r}) is below the k-th score {sk!r} but returned")


def compare(ref: RefResult, rows, scores, k):
    """Problems of one returned list (row ids, fp32 scores) against the reference; [] = accepted."""
    rows = [int(r) for r in rows]
    scores = np.asarray(scores, F32)
    problems = []
    want = min(k, len(ref.rows))
    if len(rows) != want:
        problems.append(f"count {len(rows)} != min(k, matching live documents) = {want}")
    if len(set(rows)) != len(rows):
        problems.append("duplicate rows")
    idx = []
    for j, r in enumerate(rows):
        i = ref.pos.get(r)
        if i is None:
            problems.append(f"rank {j}: row {r} is not a matching live document")
            continue
        idx.append(i)
        if abs(float(scores[j]) - ref.score[i]) > ref.tol[i]:
            problems.append(f"rank {j}: row {r} scored {float(scores[j])!r}, reference {ref.score[i]!r} +- {ref.tol[i]:.3g}")
    _kth_checks(problems, ref.score, ref.tol, np.array(idx, np.int64), want, lambda i: f"row {int(ref.rows[i])}")
    for j in range(1, len(rows)):
        if scores[j] > scores[j - 1]:
            problems.append(f"rank {j}: score {float(scores[j])!r} above the previous {float(scores[j - 1])!r}")
        elif scores[j] == scores[j - 1] and rows[j] in ref.pos and rows[j - 1] in ref.pos \
                and ref.ords[ref.pos[rows[j]]] <= ref.ords[ref.pos[rows[j - 1]]]:
            problems.append(f"rank {j}: equal scores not in ascending doc-ordinal order")
    return problems


# ---------------------------------------------------------------------------------------------------------------------
# Test corpora: tokens are the ground truth; the text the library and the oracle tokenise is rendered from them
# ---------------------------------------------------------------------------------------------------------------------
# ASCII punctuation and white space, and separators from the Unicode blocks the tokenizer documents
SEPARATORS = [" ", " ", ", ", ".", "; ", "!", " - ", "(", "\t", "\n", "，", "—", "　", "» "]


def vocabulary(n, scripts=True):
    """n distinct lowercase terms (< 40 bytes), in ASCII and, with scripts, Latin-1, Cyrillic and full-width forms."""
    out = []
    for i in range(n):
        kind = i % 4 if scripts else 0
        out.append((f"w{i}", f"été{i}", f"мир{i}", f"ｔｅｒｍ{i}")[kind])
    return out


def render(tokens, rng, mixed=True):
    """Join tokens into text with mixed separators and capitalisation (the library must lowercase them back)."""
    if not mixed:
        return " ".join(tokens)
    out = []
    for t in tokens:
        c = int(rng.integers(0, 3))
        out.append(t if c == 0 else t.upper() if c == 1 else t[:1].upper() + t[1:])
        out.append(SEPARATORS[int(rng.integers(0, len(SEPARATORS)))])
    return "".join(out)


# ---------------------------------------------------------------------------------------------------------------------
# Hybrid fusion (RankFusion / RelativeScoreFusion): entries keyed by (shard, part, label)
# ---------------------------------------------------------------------------------------------------------------------
def _normalised(scores):
    """Min / max normalisation with min = last, max = first (swapped when ascending); all equal -> 1."""
    s = np.asarray(scores, np.float64)
    if not len(s):
        return s
    mn, mx = s[-1], s[0]
    if mn == mx:
        return np.ones(len(s))
    if mn > mx:
        mn, mx = mx, mn
    return (s - mn) / (mx - mn)


def fuse(fusion_type, vec, txt, fusion_weight=0.5, fusion_k=60, vector_scan_direction=1):
    """vec / txt: lists of (shard, part, label, score), each globally ordered.  Returns {key: (score, tolerance)}.

    RRF: sum over both lists of 1 / (fusion_k + rank + 1).  RSF: text parts are ASSIGNED (a key listed twice keeps its
    last part), then vector parts are ADDED, duplicates included.  The tolerance is 1e-6 (m + 1) times the sum of the
    parts' magnitudes; for RSF a part's magnitude is its weight factor, since the normalised score it scales can lose
    an ulp of 1 in fp32 (1 - ns near ns = 1)."""
    w = float(F32(fusion_weight))
    parts = {}
    key = lambda e: (int(e[0]), int(e[1]), int(e[2]))   # noqa: E731
    if fusion_type.lower() == "rrf":
        for lst in (vec, txt):
            for i, e in enumerate(lst):
                v = 1.0 / (float(fusion_k) + i + 1)
                parts.setdefault(key(e), []).append((v, v))
    else:
        for e, ns in zip(txt, _normalised([e[3] for e in txt])):
            parts[key(e)] = [(ns * w, abs(w))]
        w1 = 1.0 - w
        for e, ns in zip(vec, _normalised([e[3] for e in vec])):
            v = (ns if vector_scan_direction == -1 else 1.0 - ns) * w1
            parts.setdefault(key(e), []).append((v, abs(w1)))
    out = {}
    for k_, ps in parts.items():
        s = sum(p[0] for p in ps)
        out[k_] = (s, 1e-6 * (len(ps) + 1) * sum(abs(p[1]) for p in ps))
    return out


def compare_fusion(ref: dict, got, top_k):
    """Problems of one fused list [(shard, part, label, fp32 score)] against fuse(); [] = accepted."""
    problems = []
    keys = list(ref)
    kidx = {k_: i for i, k_ in enumerate(keys)}
    rs = np.array([ref[k_][0] for k_ in keys])
    rt = np.array([ref[k_][1] for k_ in keys])
    want = min(top_k, len(keys))
    if len(got) != want:
        problems.append(f"count {len(got)} != min(top_k, distinct keys) = {want}")
    gk = [(int(a), int(b), int(c)) for a, b, c, _ in got]
    gs = [float(F32(e[3])) for e in got]
    if len(set(gk)) != len(gk):
        problems.append("duplicate keys")
    idx = []
    for j, (k_, s) in enumerate(zip(gk, gs)):
        i = kidx.get(k_)
        if i is None:
            problems.append(f"rank {j}: key {k_} is in neither list")
            continue
        idx.append(i)
        if abs(s - rs[i]) > rt[i]:
            problems.append(f"rank {j}: key {k_} fused to {s!r}, reference {rs[i]!r} +- {rt[i]:.3g}")
    _kth_checks(problems, rs, rt, np.array(idx, np.int64), want, lambda i: f"key {keys[i]}")
    for j in range(1, len(gk)):
        if gs[j] > gs[j - 1] or (gs[j] == gs[j - 1] and gk[j] <= gk[j - 1]):
            problems.append(f"rank {j}: not in (score descending, key ascending) order")
    return problems
