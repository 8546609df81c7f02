"""How a search reads its params string (include/b200_search.h): keys match whole words, reorder_k_factor stands for
refine_factor, a negative value of a key other than search_width reads as absent, the graph keys are checked only where the
graph is walked, and the graph's seed search takes the index's defaults at nprobe 1, never the caller's list-search keys."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from myscaledb_b200.search import B200Error

pytestmark = pytest.mark.gpu
F32 = np.float32
INVALID = 1
N, D, NQ, K = 20000, 64, 32, 10
NLIST, NPROBE = 128, 32    # NPROBE: the default nprobe of an index created without the key
REFINE = 4                 # MSTG's default refine_factor


def _clustered(seed, n_centres=200, spread=0.3):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_centres, D)).astype(F32)
    y = centres[rng.integers(0, n_centres, N)] + spread * rng.standard_normal((N, D)).astype(F32)
    q = centres[rng.integers(0, n_centres, NQ)] + spread * rng.standard_normal((NQ, D)).astype(F32)
    return y.astype(F32), q.astype(F32)


def _same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


@pytest.fixture(scope="module")
def data():
    return _clustered(3)


@pytest.fixture(scope="module")
def ivfflat(data):
    return b2.VectorIndex("IVFFLAT", b2.L2, D, f"nlist={NLIST}").build(data[0])


@pytest.fixture(scope="module")
def graphs(data):
    return {t: b2.VectorIndex(t, b2.L2, D, f"nlist={NLIST}, graph_degree=32").build(data[0]) for t in ("HNSWFLAT", "MSTG")}


def _probes(ix):
    return set(ix.last_probe()[0].tolist())


def test_keys_match_whole_words(data, ivfflat, graphs):
    q = data[1]
    base = ivfflat.search(q, K)
    assert _probes(ivfflat) == {NPROBE}
    for params in ("max_nprobe=1", "my_nprobe=1", "nprobe_x=1"):
        assert _same(ivfflat.search(q, K, params), base), f"{params!r} differs from no key"
        assert _probes(ivfflat) == {NPROBE}, f"{params!r} set nprobe"
    ivfflat.search(q, K, "nprobe=1")
    assert _probes(ivfflat) == {1}
    # "graph_degree=0" is not the key graph: the search still walks the graph
    ix = graphs["MSTG"]
    base = ix.search(q, K)
    seeds = ix.last_seeds()
    assert seeds is not None
    assert _same(ix.search(q, K, "graph_degree=0"), base)
    assert ix.last_seeds().tobytes() == seeds.tobytes()


def test_reorder_k_factor_is_refine_factor(data, graphs):
    y, q = data
    ix = b2.VectorIndex("MSTG", b2.L2, D, f"nlist={NLIST}").build(y)
    ix.search(q, K)
    assert ix.last_num_candidates == K * REFINE
    a = ix.search(q, K, "refine_factor=3")
    assert ix.last_num_candidates == 3 * K
    assert _same(ix.search(q, K, "reorder_k_factor=3"), a)
    assert ix.last_num_candidates == 3 * K
    ix.search(q, K, "refine_factor=2, reorder_k_factor=3")   # refine_factor wins
    assert ix.last_num_candidates == 2 * K
    ix.search(q, K, "reorder_k_factor=0")                    # at least 1: the first stage alone
    assert ix.last_num_candidates == K
    # the graph walk's candidates: kc = k x refine_factor
    g = graphs["MSTG"]
    g.search(q, K, "reorder_k_factor=3")
    assert g.last_num_candidates == 3 * K


def test_negative_values_read_as_absent(data, ivfflat, graphs):
    q = data[1]
    assert _same(ivfflat.search(q, K, "nprobe=-5"), ivfflat.search(q, K))
    assert _probes(ivfflat) == {NPROBE}
    for typ, ix in graphs.items():
        base = ix.search(q, K)
        seeds = ix.last_seeds()
        assert _same(ix.search(q, K, "ef_s=-5"), base), f"{typ}: ef_s=-5 differs from no key"
        assert ix.last_seeds().tobytes() == seeds.tobytes()
        # search_width alone is read signed: a negative width is refused where the walk runs
        with pytest.raises(B200Error) as e:
            ix.search(q, K, "search_width=-2")
        assert e.value.code == INVALID


def test_graph_keys_are_checked_where_the_walk_runs(data, ivfflat, graphs):
    q = data[1]
    assert _same(ivfflat.search(q, K, "ef_s=2000, search_width=3"), ivfflat.search(q, K))
    for typ, ix in graphs.items():
        assert _same(ix.search(q, K, "graph=0, ef_s=2000, search_width=3"), ix.search(q, K, "graph=0")), typ
        for params in ("ef_s=2000", "search_width=3"):
            with pytest.raises(B200Error) as e:
                ix.search(q, K, params)
            assert e.value.code == INVALID, f"{typ} {params!r}"


@pytest.mark.parametrize("typ", ["HNSWFLAT", "MSTG"])
def test_seed_search_ignores_the_callers_list_keys(data, graphs, typ):
    q = data[1]
    ix = graphs[typ]
    base = ix.search(q, K)
    seeds = ix.last_seeds()
    assert seeds is not None
    for params in ("coarse_path=1, pages_per_chunk=2, shared_bound=0", "nprobe=64"):
        got = ix.search(q, K, params)
        assert ix.last_seeds().tobytes() == seeds.tobytes(), f"{typ} {params!r}: the seeds differ"
        assert _same(got, base), f"{typ} {params!r}: the results differ"
