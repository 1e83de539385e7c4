"""CPU: boolean queries over several DataFrame fields (query.Field, solr.fields_topk) -- Field validation, flattening
to field slots, every refusal (raised before any device work, so on CPU-built arrays), and the oracle composition
against the real reference's composed results (tests/golden/bool_fields.json, make_golden_bool_fields.py)."""
import json
import os

import numpy as np
import pandas as pd
import pytest

from _bool_compose import oracle_score, topk
from _bool_fields_compose import field_scorer, query_of, record_groups
from _bool_occur_compose import compose_occur
from _tmdb_index import load_field
from conftest import GOLDEN


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "bool_fields.json")) as f:
        return json.load(f)


def frame_of(**cols):
    from searcharray_b200 import SearchArray
    return pd.DataFrame({name: SearchArray.index(docs) for name, docs in cols.items()})


def test_field_validation():
    from searcharray_b200 import And, Bool, Boost, Field, Or
    f = Field("title", "star")
    assert f.field == "title" and f.clause == "star"
    assert Field("body", ("a", "b")).clause == ["a", "b"]
    for bad in (3, [], ["a", 3], None, Boost("a", 2), Field("x", "a"), Boost(Field("x", "a"), 2)):
        with pytest.raises(TypeError):
            Field("title", bad)
    for bad in (3, None, ["title"]):
        with pytest.raises(TypeError):
            Field(bad, "star")
    b = Boost(Field("title", ["a", "b"]), 2)
    assert isinstance(b.clause, Field) and b.clause.clause == ["a", "b"] and b.weight == np.float32(2)
    # accepted wherever a clause is
    q = Or([Field("t", "a"), Boost(Field("b", "c"), 0.5)], mm=2)
    assert [c.field for c in q.clauses] == ["t", "b"] and q.weights == [1.0, 0.5] and q.mm == 2
    assert And([Field("t", "a"), Field("b", "a")]).mm == 2
    bq = Bool(must=[Field("t", "a")], should=[Boost(Field("b", "c"), 2)], filter=[Field("t", ["x", "y"])],
              must_not=[Field("b", "n")])
    assert bq.must_weights == [1.0] and bq.should_weights == [2.0] and bq.filter[0].clause == ["x", "y"]
    # Bool's and Boost's existing errors stand
    for role in ("filter", "must_not"):
        with pytest.raises(ValueError):
            Bool(should=[Field("t", "a")], **{role: [Boost(Field("b", "c"), 2)]})
    with pytest.raises(ValueError):
        Boost(Field("t", "a"), -1)
    with pytest.raises(ValueError):
        Bool(filter=[Field("t", "a")])


def test_flatten_to_field_slots():
    from searcharray_b200 import Bool, Boost, Field, Or
    from searcharray_b200.solr import _fields_plan
    fr = frame_of(t=["a b", "b c", "c"], o=["x a", "a", "y"], p=["a", "b", "c"])
    fr["t2"] = fr["t"]                            # a second name of one column: one device index, one slot
    queries = [Or([Field("o", "a"), Boost(Field("t", ["a", "b"]), 2)], mm=2),
               Bool(must=[Field("t2", "b")], should=[Field("p", "c")], filter=[Field("o", "x")],
                    must_not=[Field("t", "c")], mm=1)]
    batch, slot_of, arrays, sims = _fields_plan(fr, queries, {})
    clauses, starts, mm, weights, occurs = batch.clauses, batch.node_starts, batch.mm, batch.weights, batch.occurs
    assert batch.clause_node is None and batch.groups is None and batch.ties is None and batch.n_queries == 2
    assert [c.field for c in clauses] == ["o", "t", "t2", "p", "o", "t"]
    assert slot_of == {"o": 0, "t": 1, "t2": 1, "p": 2} and len(arrays) == 3 and len(sims) == 3
    assert arrays[1] is not None and arrays[1]._shared is fr["t2"].array._shared
    assert starts.tolist() == [0, 2, 6] and mm.tolist() == [2, 1]
    assert weights.tolist() == [1, 2, 1, 1, 1, 1] and occurs.tolist() == [0, 0, 1, 0, 2, 3]


def test_refusals():
    """Every refusal, before any device work."""
    from searcharray_b200 import Bool, Field, Or, SearchArray, bm25_impact, bm25_similarity, fields_topk
    fr = frame_of(t=["a b", "b c", "c"], o=["x a", "a", "y"])
    q = Or([Field("t", "a"), Field("o", "a")])
    with pytest.raises(ValueError, match="names its column"):
        fields_topk(fr, [Or([Field("t", "a"), "a"])])
    with pytest.raises(ValueError, match="names its column"):
        fields_topk(fr, [Bool(should=[Field("t", "a")], must_not=[["a", "b"]])])
    with pytest.raises(TypeError):
        fields_topk(fr, ["a"])
    with pytest.raises(ValueError, match="not in dataframe"):
        fields_topk(fr, [Or([Field("missing", "a")])])
    fr2 = fr.copy()
    fr2["plain"] = ["a", "b", "c"]
    with pytest.raises(ValueError, match="not a searcharray field"):
        fields_topk(fr2, [Or([Field("plain", "a")])])
    with pytest.raises(TypeError):
        fields_topk(fr, [q], similarity=bm25_impact())
    with pytest.raises(TypeError):
        fields_topk(fr, [q], similarity={"o": bm25_impact()})
    # a view among the fields
    view = pd.DataFrame({"t": fr["t"].array[np.array([True, False, True])],
                         "o": fr["o"].array[np.array([True, False, True])]})
    with pytest.raises(NotImplementedError):
        fields_topk(view, [q])
    # more than 8 distinct fields
    wide = frame_of(**{f"f{i}": ["a", "b"] for i in range(9)})
    with pytest.raises(ValueError, match="at most 8"):
        fields_topk(wide, [Or([Field(f"f{i}", "a") for i in range(9)])])
    # columns of different lengths (a mapping of Series standing in for a frame), or on different devices
    class Columns(dict):
        @property
        def columns(self):
            return list(self)
    uneven = Columns(t=pd.Series(SearchArray.index(["a", "b", "c"])), u=pd.Series(SearchArray.index(["a", "b"])))
    with pytest.raises(ValueError, match="one length"):
        fields_topk(uneven, [Or([Field("t", "a"), Field("u", "a")])])
    dev1 = pd.DataFrame({"t": fr["t"], "o": SearchArray.index(["x a", "a", "y"], device=1)})
    with pytest.raises(ValueError, match="one device"):
        fields_topk(dev1, [q])
    # one device index under two similarities
    fr3 = fr.copy()
    fr3["t2"] = fr3["t"]
    with pytest.raises(ValueError, match="shares its device index"):
        fields_topk(fr3, [Or([Field("t", "a"), Field("t2", "a")])], similarity={"t2": bm25_similarity(k1=2.0)})
    # a Field clause in SearchArray.search_topk
    with pytest.raises(ValueError, match="fields_topk"):
        fr["t"].array.search_topk([Or([Field("t", "a")])], k=2)
    with pytest.raises(ValueError, match="fields_topk"):
        fr["t"].array.search_topk(["a", Bool(should=["a"], must_not=[Field("t", "b")])], k=2)
    # none of the above touched a device
    for col in ("t", "o"):
        assert fr[col].array._shared["dev"] is None


def oracle_scorer(hosts, rec):
    from oracle import search as osearch
    out = {}
    for f, host in hosts.items():
        o = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                avg_doc_length=host.avg_doc_length)
        k1, b = rec["sim"].get(f, [1.2, 0.75])
        out[f] = oracle_score(o, host.term_dict, k1=k1, b=b, slop=rec["slop"])
    return field_scorer(out)


def test_oracle_composition_golden(fixture):
    """The oracle's per-field composition reproduces the real reference's composed top 10 (ids, score bits, n_ranked)
    of every record, and our mm parsing resolves each Solr spec as the reference's did."""
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    hosts = {f: load_field(z, f) for f in ("title_tokens", "overview_tokens")}
    recs = fixture["queries"]
    assert len(recs) >= 30
    for group in record_groups(recs).values():
        score = oracle_scorer(hosts, group[0])
        for rec in group:
            q = query_of(rec)
            assert q.mm == rec["mm"], rec["mm_spec"]
            v = compose_occur(score, q)
            ids, scores = topk(v, 10)
            n = len(rec["top_ids"])
            what = f"{q!r} slop={rec['slop']} sim={rec['sim']}"
            assert int(np.count_nonzero(v > 0)) == rec["n_ranked"], what
            assert ids[:n].tolist() == rec["top_ids"] and np.all(ids[n:] == 0xFFFFFFFF), what
            assert scores[:n].view(np.uint32).tolist() == rec["top_bits"], what
