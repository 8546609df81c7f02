"""The float64 BM25 / fusion reference (tests/bm25_reference.py) against the C oracle, and negative controls showing that
its comparator rejects the mistakes a scorer makes.  CPU only."""
import numpy as np
import pytest

import oracle as orc
from tests import bm25_reference as R

F32 = np.float32


def test_literal_fieldnorm_table_equals_the_oracle():
    assert [int(v) for v in R.FIELDNORM_TABLE] == [orc.id_to_fieldnorm(i) for i in range(256)]
    assert R.FIELDNORM_TABLE[255] == 2013265944
    lengths = list(range(0, 3000)) + [int(v) + d for v in R.FIELDNORM_TABLE for d in (-1, 0, 1) if v + d >= 0]
    assert [int(c) for c in R.fieldnorm_code(lengths)] == [orc.fieldnorm_to_id(n) for n in lengths]


def _corpus(seed, n_fields, n_docs=300):
    """Zipf tokens, Poisson lengths plus documents of 39, 40, 41, 55, 56, 1 000 and 100 000 tokens, a block of identical
    documents (real ties), sparse shuffled row ids."""
    rng = np.random.default_rng(seed)
    vocab = R.vocabulary(120)
    pz = 1.0 / np.arange(1, len(vocab) + 1) ** 1.1
    pz /= pz.sum()
    special = [39, 40, 41, 55, 56, 1000, 100000]
    docs = []
    for d in range(n_docs):
        fields = []
        for f in range(n_fields):
            ln = special[d % len(special)] if (d < 3 * len(special) and d % n_fields == f) else int(rng.poisson(12))
            if f == 1 and d % 17 == 0:
                ln = 0   # empty field
            fields.append([str(t) for t in rng.choice(vocab, size=ln, p=pz)])
        docs.append(fields)
    for d in range(n_docs - 6, n_docs):
        docs[d] = [list(x) for x in docs[n_docs - 7]]
    rows = rng.choice(1 << 20, size=n_docs, replace=False)
    return docs, rows, vocab, rng


def _both(docs, rows, rng, n_fields):
    o = orc.BM25Index(n_fields)
    for fields, r in zip(docs, rows):
        o.add_doc(int(r), [R.render(t, rng) for t in fields])
    return o, R.BM25Reference.from_tokens(docs, rows)


def _queries(vocab, rng):
    qs = [[vocab[i] for i in rng.integers(0, 40, size=int(rng.integers(1, 6)))] for _ in range(24)]
    qs += [[vocab[0]], [vocab[0], vocab[1], vocab[2]], [vocab[100], "nosuchterm"], ["nosuchterm"], [vocab[3]] * 4,
           vocab[:70]]
    return qs


@pytest.mark.parametrize("n_fields,fields", [(1, (0,)), (2, (0, 1)), (2, (1,)), (3, (0, 1, 2)), (3, (2, 0))])
@pytest.mark.parametrize("operator_or", [True, False])
@pytest.mark.parametrize("table_stats", [False, True])
def test_reference_agrees_with_the_oracle(n_fields, fields, operator_or, table_stats):
    docs, rows, vocab, rng = _corpus(5 + n_fields, n_fields)
    o, ref = _both(docs, rows, rng, n_fields)
    assert [o.doc_len(d, f) for d in range(len(docs)) for f in range(n_fields)] == \
           [len(docs[d][f]) for d in range(len(docs)) for f in range(n_fields)]
    stats = None
    if table_stats:   # this part plus others the part has never seen
        st = ref.stats()
        stats = dict(total_docs=st["total_docs"] + 5000, total_tokens={f: v + 61000 for f, v in st["total_tokens"].items()},
                     doc_freq={key: v + 7 * (len(key[1]) % 5) for key, v in st["doc_freq"].items()})
    alive = rng.random(int(rows.max()) + 1) < 0.7
    for qi, q in enumerate(_queries(vocab, rng)):
        sentence = R.render(q, rng)
        for k, al in ((10, None), (400, alive)):
            got_rows, got_scores = o.search(sentence, k, fields=fields, operator_or=operator_or, stats=stats,
                                            alive=None if al is None else orc.pack_bits(al))
            want = ref.search(q, fields=fields, alive=al, operator_or=operator_or, stats=stats)
            problems = R.compare(want, got_rows, got_scores, k)
            assert not problems, (qi, q[:5], k, problems[:5])


def _rsf_rrf_lists(rng, nv, nt, big):
    """Candidate lists with duplicate keys inside one list and keys at the top of their ranges."""
    shard_vals = [0, 1, 2 ** 32 - 1] if big else [0, 1]
    part_vals = [0, 3, 2 ** 63] if big else [0, 3]
    label_vals = [2 ** 53, 2 ** 53 + 1, 2 ** 53 + 3, 2 ** 63, 2 ** 64 - 1, 2 ** 64 - 2, 7, 8] if big else list(range(8))

    def one(n, desc):
        sc = np.sort(rng.random(n).astype(F32))
        if desc:
            sc = sc[::-1]
        keys = [(shard_vals[rng.integers(len(shard_vals))], part_vals[rng.integers(len(part_vals))],
                 label_vals[rng.integers(len(label_vals))]) for _ in range(n)]
        return [(a, b, c, float(s)) for (a, b, c), s in zip(keys, sc)]
    return one(nv, False), one(nt, True)


@pytest.mark.parametrize("ft", ["rrf", "rsf"])
@pytest.mark.parametrize("direction", [1, -1])
@pytest.mark.parametrize("big", [False, True])
def test_fusion_reference_agrees_with_the_oracle(ft, direction, big):
    rng = np.random.default_rng(31 + direction + 2 * big)
    for trial in range(60):
        vec, txt = _rsf_rrf_lists(rng, int(rng.integers(0, 12)), int(rng.integers(0, 12)), big)
        if direction == -1:
            vec = vec[::-1]
        if trial % 9 == 0 and vec:
            vec = [(a, b, c, vec[0][3]) for a, b, c, _ in vec]   # all equal: normalised to 1
        for top_k, w, fk in ((5, 0.3, 60), (100, 0.0, 0), (3, 1.0, 2 ** 40)):
            got = orc.hybrid_fusion(ft, vec, txt, top_k, fusion_weight=w, fusion_k=fk, vector_scan_direction=direction)
            want = R.fuse(ft, vec, txt, fusion_weight=w, fusion_k=fk, vector_scan_direction=direction)
            problems = R.compare_fusion(want, got, top_k)
            assert not problems, (trial, top_k, w, fk, problems[:5])


# ---- negative controls: each mistake must be rejected by the comparator
def _control_corpus():
    rng = np.random.default_rng(77)
    vocab = R.vocabulary(30, scripts=False)
    docs = [[[str(t) for t in rng.choice(vocab[:20], size=int(rng.integers(5, 30)))]] for _ in range(200)]
    docs[10] = [[vocab[25]] * 3 + [vocab[0]] * 40]            # 43 tokens: code 41 stands for 42
    docs[11] = [[vocab[25]] * 2 + [vocab[1]] * 10]
    docs[12] = [[vocab[26], vocab[2], vocab[3]]]
    docs[13] = [[vocab[26], vocab[2], vocab[3]]]               # identical to doc 12: a real tie
    return docs, vocab, R.BM25Reference.from_tokens(docs, np.arange(200) * 3 + 1)


def test_comparator_accepts_the_expected_list():
    docs, vocab, ref = _control_corpus()
    for q in ([vocab[25]], [vocab[26]], [vocab[25], vocab[2]], [vocab[0]]):
        want = ref.search(q)
        rows, scores = want.topk(5)
        assert not R.compare(want, rows, scores, 5)


def test_comparator_rejects_the_raw_length_instead_of_its_code():
    docs, vocab, ref = _control_corpus()
    assert len(docs[10][0]) == 43 and R.FIELDNORM_TABLE[R.fieldnorm_code(43)] == 42
    raw = R.BM25Reference.from_tokens(docs, ref.row_ids, quantise_lengths=False)
    rows, scores = raw.search([vocab[25]]).topk(5)
    assert ref.row_ids[10] in rows.tolist()
    assert R.compare(ref.search([vocab[25]]), rows, scores, 5)


def test_comparator_rejects_a_dropped_posting():
    docs, vocab, ref = _control_corpus()
    q = [vocab[25], vocab[2]]
    want = ref.search(q)
    rows, scores = want.topk(10)
    docs_c, contrib = ref.clause_contributions(0, vocab[25])
    assert contrib.max() > 1   # a term with idf > 1
    i = list(rows).index(ref.row_ids[docs_c[0]])
    bad = scores.astype(np.float64)
    bad[i] -= contrib[0]
    order = np.argsort(-bad, kind="stable")
    assert R.compare(want, rows[order], bad[order].astype(F32), 10)


def test_comparator_rejects_a_wrong_tie_order():
    docs, vocab, ref = _control_corpus()
    want = ref.search([vocab[26]])
    rows, scores = want.topk(5)
    assert len(rows) == 2 and scores[0] == scores[1]
    assert not R.compare(want, rows, scores, 5)
    assert R.compare(want, rows[::-1], scores[::-1], 5)


def test_comparator_rejects_a_missing_last_result():
    docs, vocab, ref = _control_corpus()
    want = ref.search([vocab[0]])
    rows, scores = want.topk(20)
    assert len(rows) == 20
    assert R.compare(want, rows[:-1], scores[:-1], 20)


def test_fusion_comparator_rejects_a_wrong_key_and_a_wrong_sum():
    vec = [(0, 0, 2 ** 53 + 1, 0.1), (0, 0, 5, 0.2), (0, 0, 5, 0.3)]
    txt = [(0, 0, 5, 9.0), (0, 0, 2 ** 53 + 1, 4.0), (0, 0, 7, 1.0)]
    want = R.fuse("rsf", vec, txt, fusion_weight=0.3)
    got = orc.hybrid_fusion("rsf", vec, txt, 10, fusion_weight=0.3)
    assert not R.compare_fusion(want, got, 10)
    rounded = [(a, b, 2 ** 53 if c == 2 ** 53 + 1 else c, s) for a, b, c, s in got]
    assert R.compare_fusion(want, rounded, 10)
    # the vector part of the duplicated vector key added once only
    once = R.fuse("rsf", vec[:2], txt, fusion_weight=0.3)
    assert R.compare_fusion(want, sorted(((*k, F32(v[0])) for k, v in once.items()), key=lambda e: (-e[3], e[:3])), 10)
