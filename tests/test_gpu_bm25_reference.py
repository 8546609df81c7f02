"""BM25 text search and hybrid fusion on the GPU at production shapes.  Every case feeds the same generated documents to the
GPU index, the C oracle and the float64 reference (tests/bm25_reference.py), and checks that the GPU is bit-identical to the
oracle and accepted by the reference's comparator.  The corpora reach the cases the toy-sized parity tests never do: several
CTAs per query and ranges the DAAT kernel must halve and widen again, 64-clause queries, k up to 2048, documents long
enough for the 1-byte field-norm code to quantise their length, row ids in another order than the doc ordinals (ties go to
the smaller ordinal), batches above gridDim.y, and fusion lists with duplicate keys and 64-bit labels."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from tests import bm25_reference as R

pytestmark = pytest.mark.gpu
F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Corpus:
    """One set of documents in the GPU index, the oracle and the reference."""

    def __init__(self, vocab, fields, row_ids, texts):
        self.vocab, self.row_ids = vocab, np.asarray(row_ids, np.int64)
        self.n_fields = len(fields)
        self.gpu, self.orc = b2.BM25Index(self.n_fields), orc.BM25Index(self.n_fields)
        for d, r in enumerate(self.row_ids.tolist()):
            t = [texts[f][d] for f in range(self.n_fields)]
            self.gpu.add_doc(r, t)
            self.orc.add_doc(r, t)
        self.gpu.commit()
        self.ref = R.BM25Reference(vocab, fields, row_ids)

    @classmethod
    def from_tokens(cls, docs, row_ids, rng):
        ref = R.BM25Reference.from_tokens(docs, row_ids)
        n_fields = len(docs[0]) if docs else 1
        fields = [(np.concatenate([[0], np.cumsum([len(d[f]) for d in docs])]).astype(np.int64),
                   np.array([ref.term_id[t] for d in docs for t in d[f]], np.int64)) for f in range(n_fields)]
        texts = [[R.render(d[f], rng) for d in docs] for f in range(n_fields)]
        return cls(ref.vocab, fields, row_ids, texts)

    def check(self, queries, k, fields=(0,), alive=None, operator_or=True, stats=None, ref_every=1, gpu=None):
        """queries: token lists.  GPU == oracle bit for bit on every query; the reference accepts every ref_every-th."""
        sentences = [" ".join(q) for q in queries]
        ab = None if alive is None else orc.pack_bits(alive)
        got = gpu if gpu is not None else self.gpu.search_batch(sentences, k, fields=fields, alive_bits=ab,
                                                                 operator_or=operator_or, stats=stats)
        for qi, (q, s) in enumerate(zip(queries, sentences)):
            rows, scores = got[qi]
            orow, oscore = self.orc.search(s, k, fields=fields, alive=ab, operator_or=operator_or, stats=stats)
            assert rows.tolist() == orow.tolist() and scores.view(np.uint32).tolist() == oscore.view(np.uint32).tolist(), \
                (qi, q[:4], k, fields, operator_or)
            if qi % ref_every == 0:
                want = self.ref.search(q, fields=fields, alive=alive, operator_or=operator_or, stats=stats)
                problems = R.compare(want, rows, scores, k)
                assert not problems, (qi, q[:4], k, problems[:4])
        return got


def _sparse_rows(rng, n):
    """Distinct row ids below 2^27, shuffled: tie order (by ordinal) differs from row-id order."""
    return rng.choice(1 << 27, size=n, replace=False)


@pytest.fixture(scope="module")
def zipf():
    """~300k documents, vocabulary 20k, log-normal lengths 1..2000: common terms have df far above 100k, so several CTAs
    share one query and their ranges are merged across blocks; the last 41 documents are identical (real ties)."""
    rng = np.random.default_rng(2024)
    n, nv = 300_000, 20_000
    vocab = R.vocabulary(nv, scripts=False)
    lens = np.clip(np.rint(rng.lognormal(2.6, 1.0, n)), 1, 2000).astype(np.int64)
    lens[-40:] = lens[-41]
    pz = 1.0 / np.arange(1, nv + 1) ** 1.05
    ids = rng.choice(nv, size=int(lens.sum()), p=pz / pz.sum())
    offsets = np.concatenate([[0], np.cumsum(lens)])
    vocab.append("tieblock")   # a term of the 41 identical documents only
    ids[offsets[n - 41]] = nv
    for d in range(n - 40, n):
        ids[offsets[d]:offsets[d + 1]] = ids[offsets[n - 41]:offsets[n - 40]]
    va = np.array(vocab)
    texts = [" ".join(va[ids[offsets[d]:offsets[d + 1]]]) for d in range(n)]
    c = Corpus(vocab, [(offsets, ids)], _sparse_rows(rng, n), [texts])
    c.pz = pz / pz.sum()
    c.lens, c.offsets, c.ids = lens, offsets, ids
    return c


def _zipf_queries(c, rng, nq, lo=1, hi=5):
    return [[c.vocab[i] for i in rng.choice(len(c.pz), size=int(rng.integers(lo, hi + 1)), p=c.pz)] for _ in range(nq)]


@pytest.mark.parametrize("k,nq,operator_or,alive_frac", [
    (1, 1, True, 1.0), (31, 8, True, 0.5), (32, 8, False, 1.0), (33, 8, True, 0.01), (100, 1, True, 0.0),
    (257, 8, False, 0.5), (1024, 8, True, 1.0), (2048, 1, True, 0.5), (100, 591, True, 1.0), (32, 592, False, 0.5),
    (33, 593, True, 1.0), (10, 2000, True, 0.5)])
def test_zipf_corpus(zipf, k, nq, operator_or, alive_frac):
    rng = np.random.default_rng(k * 7 + nq)
    queries = _zipf_queries(zipf, rng, nq)
    queries[0] = [zipf.vocab[0], zipf.vocab[1], zipf.vocab[2]]   # the three most common terms
    queries[-1] = list(zipf.ref.vocab[i] for i in zipf.ids[zipf.offsets[-41]:zipf.offsets[-40]][:3])   # hits the tie block
    alive = None
    if alive_frac < 1.0:
        alive = np.zeros(int(zipf.row_ids.max()) + 1, bool)
        alive[zipf.row_ids] = rng.random(len(zipf.row_ids)) < alive_frac
    zipf.check(queries, k, alive=alive, operator_or=operator_or, ref_every=max(1, nq // 40))


def test_zipf_ties_go_to_the_smaller_ordinal(zipf):
    rows, scores = zipf.check([["tieblock"]], 64)[0]
    assert len(rows) == 41 and len(set(scores.tolist())) == 1
    assert rows.tolist() == zipf.row_ids[-41:].tolist()   # ordinal order, not row-id order
    assert sorted(rows.tolist()) != rows.tolist()


def test_zipf_batch_order_repeat_and_single_queries_agree(zipf):
    rng = np.random.default_rng(5)
    qs = [" ".join(q) for q in _zipf_queries(zipf, rng, 24, 1, 8)]
    a = zipf.gpu.search_batch(qs, 100)
    b = zipf.gpu.search_batch(qs, 100)
    c = zipf.gpu.search_batch(qs[::-1], 100)[::-1]
    d = [zipf.gpu.search(s, 100) for s in qs]
    for x in (b, c, d):
        for (r0, s0), (r1, s1) in zip(a, x):
            assert r0.tobytes() == r1.tobytes() and s0.tobytes() == s1.tobytes()


_TAAT_SCRIPT = textwrap.dedent("""
    import json, sys
    sys.path.insert(0, sys.argv[1])
    import numpy as np
    import myscaledb_b200 as b2
    spec = json.load(open(sys.argv[2]))
    ix = b2.BM25Index.load(spec["index"], spec["n_fields"])
    out = {}
    for i, case in enumerate(spec["cases"]):
        res = ix.search_batch(case["queries"], case["k"], fields=tuple(case["fields"]), operator_or=case["or"])
        out[f"r{i}"] = np.concatenate([r for r, _ in res] + [np.zeros(0, np.uint64)])
        out[f"s{i}"] = np.concatenate([s for _, s in res] + [np.zeros(0, np.float32)])
        out[f"c{i}"] = np.array([len(r) for r, _ in res])
    ix.close()
    np.savez(spec["out"], **out)
""")


def _taat_equals_daat(c, cases, tmp_path):
    """The round-1 term-at-a-time kernel (B200_BM25_TAAT=1, read once per process: a subprocess over the saved index) and the
    default DAAT kernel give byte-identical results."""
    import json
    idx, spec_p, out_p = tmp_path / "ix.b2tx", tmp_path / "spec.json", tmp_path / "taat.npz"
    c.gpu.save(idx)
    spec_p.write_text(json.dumps(dict(index=str(idx), n_fields=c.n_fields, out=str(out_p), cases=[
        dict(queries=q, k=k, fields=list(f), **{"or": o}) for q, k, f, o in cases])))
    env = dict(os.environ, B200_BM25_TAAT="1")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _TAAT_SCRIPT, ROOT, str(spec_p)], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    taat = np.load(out_p)
    for i, (q, k, f, o) in enumerate(cases):
        res = c.gpu.search_batch(q, k, fields=f, operator_or=o)
        assert taat[f"c{i}"].tolist() == [len(x) for x, _ in res]
        assert taat[f"r{i}"].tobytes() == np.concatenate([x for x, _ in res] + [np.zeros(0, np.uint64)]).tobytes()
        assert taat[f"s{i}"].tobytes() == np.concatenate([s for _, s in res] + [np.zeros(0, np.float32)]).tobytes()


def test_zipf_taat_equals_daat_and_save_load(zipf, tmp_path):
    rng = np.random.default_rng(8)
    qs = [" ".join(q) for q in _zipf_queries(zipf, rng, 40, 1, 6)]
    _taat_equals_daat(zipf, [(qs[:1], 2048, (0,), True), (qs, 100, (0,), True), (qs, 33, (0,), False)], tmp_path)
    loaded = b2.BM25Index.load(tmp_path / "ix.b2tx", 1)
    for (r0, s0), (r1, s1) in zip(zipf.gpu.search_batch(qs, 257), loaded.search_batch(qs, 257)):
        assert r0.tobytes() == r1.tobytes() and s0.tobytes() == s1.tobytes()
    loaded.close()


@pytest.fixture(scope="module")
def dense():
    """20k documents over 2 fields; ordinals 5000..6999 hold all 32 hot terms in both fields (64 clauses), which are rare
    elsewhere.  The host picks a wide range for such a query; the hot run overflows the posting table again and again (the
    range is halved) and the kernel must widen the range once the run is passed."""
    rng = np.random.default_rng(11)
    n = 20_000
    vocab = R.vocabulary(400)
    hot = vocab[:33]
    docs = []
    for d in range(n):
        fields = []
        for f in range(2):
            toks = [vocab[i] for i in rng.integers(33, 400, size=int(rng.integers(3, 25)))]
            if 5000 <= d < 7000:
                toks += hot[:32] + [hot[32]] * (d % 3)
            elif rng.random() < 0.02:
                toks += [hot[int(rng.integers(0, 33))]]
            rng.shuffle(toks)
            fields.append(toks)
        docs.append(fields)
    c = Corpus.from_tokens(docs, _sparse_rows(rng, n), rng)
    c.hot = hot
    return c


@pytest.mark.parametrize("k", [1, 32, 100, 2048])
def test_dense_run_64_clauses(dense, k):
    hot = dense.hot
    queries = [hot[:32], hot[:32][::-1], hot[:5] + ["unknownterm"], hot[31:32] * 3, hot[1:33]]
    for fields in ((0, 1), (1,), (1, 0)):
        for op in (True, False):
            dense.check(queries + ([hot] if len(fields) == 1 else []), k, fields=fields, operator_or=op)
    with pytest.raises(b2.B200Error) as e:   # 33 terms x 2 fields = 66 clauses
        dense.gpu.search(" ".join(hot[:33]), 10, fields=(0, 1))
    assert e.value.code == 3


def test_dense_run_taat_equals_daat(dense, tmp_path):
    hot = dense.hot
    qs = [" ".join(hot[:32]), " ".join(hot[:7]), hot[3], " ".join(hot[10:30])]
    _taat_equals_daat(dense, [(qs, 2048, (0, 1), True), (qs, 100, (0, 1), False), (qs, 32, (1,), True)], tmp_path)


def test_tiny_and_degenerate_corpora():
    rng = np.random.default_rng(3)
    vocab = R.vocabulary(80)
    empty = Corpus.from_tokens([], [], rng)
    empty.check([[vocab[0], vocab[1]]], 10)
    one = Corpus.from_tokens([[[vocab[0], vocab[1], vocab[0]], []]], [7], rng)
    one.check([[vocab[0]], [vocab[1], vocab[0]], []], 5, fields=(0, 1))
    docs = [[[vocab[i] for i in rng.integers(0, 80, size=int(rng.integers(0, 9)))],
             [vocab[i] for i in rng.integers(0, 80, size=int(rng.integers(0, 3)))]] for _ in range(211)]
    c = Corpus.from_tokens(docs, _sparse_rows(rng, 211), rng)
    queries = [[], ["nosuchterm"], ["nosuch", "unknown"], [vocab[4]] * 5, [vocab[2], vocab[9]], vocab[:20]]
    for fields in ((0,), (1,), (0, 1)):
        long = [vocab[:63], vocab[:64], vocab[:65]] if len(fields) == 1 else []   # 63 / 64 / 65 distinct terms
        for op in (True, False):
            for k in (1, 33, 300):
                c.check(queries + long, k, fields=fields, operator_or=op)
    with pytest.raises(b2.B200Error) as e:   # 64 terms known in both fields: more than 64 clauses
        c.gpu.search(" ".join(vocab[:64]), 10, fields=(0, 1))
    assert e.value.code == 3
    for s in ("", ",;!? — 　，", "nosuchterm"):
        assert [len(r) for r, _ in c.gpu.search_batch([s], 10)] == [0]
    for bad_k in (0, 2049):
        with pytest.raises(b2.B200Error) as e:
            c.gpu.search("w0", bad_k)
        assert e.value.code == 3


def test_long_documents_and_every_code_boundary(tmp_path):
    """One term repeated 100 000 times, and documents of every length from 39 to 60 tokens, where the field-norm code
    stands for a shorter length."""
    rng = np.random.default_rng(4)
    vocab = R.vocabulary(30)
    docs = [[[vocab[0]] * 100_000]]
    for ln in range(39, 61):
        for rep in range(3):
            docs.append([[vocab[1]] * (1 + rep) + [vocab[int(i)] for i in rng.integers(2, 30, size=ln - 1 - rep)]])
    c = Corpus.from_tokens(docs, _sparse_rows(rng, len(docs)), rng)
    qs = [[vocab[0]], [vocab[1]], [vocab[1], vocab[0]], [vocab[5], vocab[1]], vocab[:30]]
    for op in (True, False):
        c.check(qs, 100, operator_or=op)
    _taat_equals_daat(c, [([" ".join(q) for q in qs], 100, (0,), True)], tmp_path)


def test_table_wide_statistics_over_three_parts_equal_one_index():
    rng = np.random.default_rng(12)
    vocab = R.vocabulary(300)
    pz = 1.0 / np.arange(1, 301) ** 1.1
    pz /= pz.sum()
    docs = [[[str(t) for t in rng.choice(vocab, size=int(rng.integers(1, 60)), p=pz)] for _ in range(3)] for _ in range(6000)]
    rows = _sparse_rows(rng, 6000)
    whole = Corpus.from_tokens(docs, rows, rng)
    cuts = [0, 1500, 4200, 6000]
    parts = [Corpus.from_tokens(docs[a:b], rows[a:b], rng) for a, b in zip(cuts, cuts[1:])]
    st = whole.ref.stats()
    assert st["total_docs"] == sum(p.gpu.total_docs for p in parts)
    assert all(st["total_tokens"][f] == sum(p.gpu.total_tokens(f) for p in parts) for f in range(3))
    queries = [[str(t) for t in rng.choice(vocab, size=int(rng.integers(1, 5)), p=pz)] for _ in range(30)]
    for fields in ((0, 1, 2), (2,), (0, 2)):
        for op in (True, False):
            want = whole.check(queries, 50, fields=fields, operator_or=op)
            per_part = [p.check(queries, 50, fields=fields, operator_or=op, stats=st) for p in parts]
            for qi in range(len(queries)):
                sc, pa, la = [], [], []
                for pi, res in enumerate(per_part):
                    sc += res[qi][1].tolist(); pa += [pi] * len(res[qi][1]); la += res[qi][0].astype(np.int64).tolist()
                s, _, lab = orc.merge_parts(sc, pa, la, 50, desc=True)
                ws, wr = want[qi][1], want[qi][0]
                assert s.tobytes() == ws.tobytes(), (qi, fields, op)
                if len(s):   # equal scores may come in another order from the merge; the rows above the last score may not
                    top = s > s[-1]
                    assert sorted(lab[top].tolist()) == sorted(wr[top].astype(np.int64).tolist())


def test_batch_above_grid_limit():
    """65 553 queries in one call: more than gridDim.y (65 535) holds, so the scoring kernel runs in slices."""
    rng = np.random.default_rng(21)
    vocab = R.vocabulary(200)
    docs = [[[vocab[int(i)] for i in rng.integers(0, 200, size=int(rng.integers(1, 20)))]] for _ in range(1500)]
    c = Corpus.from_tokens(docs, _sparse_rows(rng, 1500), rng)
    queries = [[vocab[int(i)] for i in rng.integers(0, 200, size=int(rng.integers(1, 4)))] for _ in range(65_553)]
    got = c.check(queries, 8, ref_every=997)
    assert sum(len(r) for r, _ in got[65_535:]) > 0


def test_long_sentence_with_statistics():
    """A sentence of 200 distinct 30-byte terms with table-wide statistics: the search uses the first 64."""
    rng = np.random.default_rng(9)
    terms = [f"t{i:03d}" + "x" * 26 for i in range(200)]
    docs = [[[terms[int(i)] for i in rng.integers(0, 200, size=12)]] for _ in range(500)]
    c = Corpus.from_tokens(docs, _sparse_rows(rng, 500), rng)
    st = c.ref.stats()
    st = dict(total_docs=st["total_docs"] * 3, total_tokens={0: st["total_tokens"][0] * 3},
              doc_freq={kk: v * 3 for kk, v in st["doc_freq"].items()})
    assert len(b2.BM25Index.query_terms(" ".join(terms))) == 200
    for op in (True, False):
        c.check([terms, terms[::-1], terms[100:]], 100, stats=st, operator_or=op)


# ---------------------------------------------------------------------------------------------------------------------
# Hybrid fusion
# ---------------------------------------------------------------------------------------------------------------------
_SHARDS = [0, 1, 2 ** 32 - 1]
_PARTS = [0, 5, 2 ** 63, 2 ** 64 - 1]
_LABELS = [0, 3, 2 ** 32 - 1, 2 ** 53 + 1, 2 ** 63, 2 ** 64 - 1]


def _fusion_lists(rng, nq, nv_max, nt_max, desc_vec=False, equal=False, n_keys=12, exact=False):
    keys = [(_SHARDS[i % 3], _PARTS[(i // 3) % 4], _LABELS[(i // 12) % 6] + i) if i < 72 else (0, 0, i)
            for i in range(max(n_keys, 1))]
    keys = [(a, b, min(c, 2 ** 64 - 1)) for a, b, c in keys]

    def one(n, desc):
        sc = np.sort(rng.random(n).astype(F32))
        if desc:
            sc = sc[::-1]
        if equal and n:
            sc[:] = sc[0]
        pick = rng.integers(0, len(keys), size=n)   # duplicate keys inside one list are likely
        return [(*keys[j], float(s)) for j, s in zip(pick, sc)]
    vec = [one(nv_max if exact else int(rng.integers(0, nv_max + 1)), desc_vec) for _ in range(nq)]
    txt = [one(nt_max if exact else int(rng.integers(0, nt_max + 1)), True) for _ in range(nq)]
    return vec, txt


def _check_fusion(ft, vec, txt, top_k, w, fk, direction, ref_every=1):
    got = b2.hybrid_fusion_batch(ft, vec, txt, top_k, fusion_weight=w, fusion_k=fk, vector_scan_direction=direction)
    for q in range(len(vec)):
        exp = orc.hybrid_fusion(ft, vec[q], txt[q], top_k, fusion_weight=w, fusion_k=fk, vector_scan_direction=direction)
        assert [(a, b, c, F32(d).view(np.uint32)) for a, b, c, d in got[q]] == \
               [(a, b, c, F32(d).view(np.uint32)) for a, b, c, d in exp], (ft, q, top_k, w, fk, direction)
        if q % ref_every == 0:
            problems = R.compare_fusion(R.fuse(ft, vec[q], txt[q], w, fk, direction), got[q], top_k)
            assert not problems, (ft, q, problems[:4])


@pytest.mark.parametrize("ft", ["rsf", "rrf"])
@pytest.mark.parametrize("direction", [1, -1])
def test_fusion_duplicates_wide_keys_and_weights(ft, direction):
    rng = np.random.default_rng(40 + direction)
    for nq, top_k, w, fk, equal in ((1, 1, 0.3, 60, False), (513, 10, 0.0, 0, False), (513, 10, 1.0, 2 ** 40, True),
                                    (513, 100, 0.3, 60, False)):
        vec, txt = _fusion_lists(rng, nq, 24, 24, desc_vec=direction == -1, equal=equal)
        vec[0], txt[0] = vec[0][:1], []   # one side only, a single entry
        _check_fusion(ft, vec, txt, top_k, w, fk, direction)


def test_fusion_100k_queries_in_one_call():
    rng = np.random.default_rng(41)
    vec, txt = _fusion_lists(rng, 100_000, 6, 6)
    for ft in ("rsf", "rrf"):
        _check_fusion(ft, vec, txt, 10, 0.3, 60, 1, ref_every=211)


@pytest.mark.parametrize("nv,nt", [(1, 1), (1024, 1024), (2047, 1)])
def test_fusion_strides_up_to_2048(nv, nt):
    """A total stride of 2048 needs 64 KB of shared memory, above the 48 KB default."""
    rng = np.random.default_rng(nv + nt)
    for ft in ("rsf", "rrf"):
        vec, txt = _fusion_lists(rng, 3, nv, nt, n_keys=3000, exact=True)
        for top_k in (1, 2048, 5000):
            _check_fusion(ft, vec, txt, top_k, 0.3, 60, 1)
    with pytest.raises(b2.B200Error) as e:
        b2.hybrid_fusion_batch("rrf", [[(0, 0, i, 0.0) for i in range(2048)]], [[(0, 0, 1, 1.0)]], 10)
    assert e.value.code == 3


def test_end_to_end_bm25_flat_fusion(zipf):
    """BM25 top-100 on the Zipf corpus plus FLAT top-100, fused by RSF and by RRF: bit-identical to the oracle chain."""
    rng = np.random.default_rng(6)
    n = 1000   # vector rows for the first 1000 documents; L2 distances (2p - 0.5)^2 are exact and distinct
    y = np.zeros((n, 4), F32)
    y[:, 0] = 2 * rng.permutation(n)
    x = np.array([[0.5, 0, 0, 0]], F32)
    dg, ig = b2.part_scan(b2.L2, x, y, 100)
    do, io = orc.part_scan(orc.L2, x, y, 100)
    assert ig.tolist() == io.tolist() and dg.tobytes() == do.tobytes()
    vec = [(0, 0, int(zipf.row_ids[i]), float(d)) for i, d in zip(ig[0], dg[0])]
    sentence = " ".join([zipf.vocab[3], zipf.vocab[50], zipf.vocab[700]])
    rows, sc = zipf.gpu.search(sentence, 100)
    orow, osc = zipf.orc.search(sentence, 100)
    assert rows.tolist() == orow.tolist() and sc.tobytes() == osc.tobytes()
    txt = [(0, 0, int(r), float(s)) for r, s in zip(rows, sc)]
    for ft in ("rsf", "rrf"):
        _check_fusion(ft, [vec], [txt], 100, 0.5, 60, 1)
