"""Boolean-query fixture: the reference's own and/or scenarios, and multi-clause queries on the TMDB corpus
composed through the REAL reference the way its tests compose them (test/test_search.py:126-226):

    scores = arr.score(c0) + arr.score(c1) + ...                          float32, clause order
    ok     = np.sum(np.array([arr.score(c) for c in clauses]) > 0, axis=0) >= mm

    python tests/golden/make_golden_bool.py      (build container only)

Writes tests/golden/bool_scenarios.json: the and_scenarios / or_scenarios tables (docs, clauses, mm, expected
masks; read from the imported test module, no reference source copied) and, per TMDB query, the top 10 of
np.where(ok, scores, 0) by (score desc, id asc) over scores > 0: ids and float32 score bits.
"""
import json
import os
import sys

import numpy as np

from make_golden import import_reference, HERE, SCRATCH
from make_golden_scenarios import period_compress
from make_golden_tmdb import load_corpus

# (field, clauses, mm): terms of every df bucket, phrases, duplicates, unknown tokens, mm from 0 to all clauses
TMDB_QUERIES = [
    ("title_tokens", ["Star", "Wars"], 1), ("title_tokens", ["Star", "Wars"], 2),
    ("title_tokens", ["the", "of", "a"], 1), ("title_tokens", ["the", "of", "a"], 2),
    ("title_tokens", ["the", "of", "a"], 3), ("title_tokens", ["Black", ["Star", "Wars"]], 1),
    ("title_tokens", [["Star", "Wars"], "Empire", "Strikes"], 2), ("title_tokens", ["Star", "Star", "Trek"], 1),
    ("title_tokens", ["zzzzunknown", "Mirror:"], 1), ("title_tokens", ["zzzzunknown", "qqqqunknown"], 0),
    ("title_tokens", ["The", "the", "of", "and", "A", "in"], 2), ("title_tokens", [["of", "the"], "Lord", "Rings"], 2),
    ("overview_tokens", ["war", "love", "family"], 1), ("overview_tokens", ["war", "love", "family"], 2),
    ("overview_tokens", ["the", "a", "of", "to", "and"], 5), ("overview_tokens", ["young", ["New", "York"]], 2),
    ("overview_tokens", [["in", "the"], "city", "police"], 1), ("overview_tokens", ["galactic", "empire", "rebel"], 0),
    ("overview_tokens", ["murder", "detective", "mystery", "killer"], 2), ("overview_tokens", ["the", "the"], 1),
]


def composed(arr, clauses, mm):
    scores = [arr.score(c) for c in clauses]
    s = scores[0]
    for v in scores[1:]:
        s = s + v
    ok = np.sum(np.array(scores) > 0, axis=0) >= mm
    return np.where(ok, s, np.float32(0)).astype(np.float32), ok


def top10(v):
    order = np.lexsort((np.arange(len(v)), -v.astype(np.float64)))[:10]
    order = order[v[order] > 0]
    return [int(i) for i in order], [int(b) for b in v[order].view(np.uint32)]


def main():
    import_reference()
    sys.path.insert(0, os.path.join(SCRATCH, "test"))
    from searcharray.postings import SearchArray
    captured = []
    real_index = SearchArray.index.__func__

    def capturing_index(cls, array, *a, **kw):
        captured.append(list(array))
        return real_index(cls, array, *a, **kw)
    SearchArray.index = classmethod(capturing_index)
    import test_search as ts
    out = {"and": [], "or": [], "tmdb": []}
    for kind, table in (("and", ts.and_scenarios), ("or", ts.or_scenarios)):
        for name, sc in table.items():
            captured.clear()
            arr = sc["docs"]()
            clauses = [list(c) if isinstance(c, list) else c for c in sc["keywords"]]
            mm = len(clauses) if kind == "and" else sc["min_should_match"]
            v, ok = composed(arr, clauses, mm)
            assert np.array_equal(ok, np.asarray(sc["expected"])), name
            ids, bits = top10(v)
            out[kind].append({"name": name, "docs": period_compress(captured[-1]), "clauses": clauses, "mm": mm,
                              "expected": period_compress([bool(x) for x in sc["expected"]]),
                              "top_ids": ids, "top_bits": bits})
    SearchArray.index = classmethod(real_index)
    titles, overviews = load_corpus()
    arrs = {"title_tokens": SearchArray.index(titles), "overview_tokens": SearchArray.index(overviews)}
    for field, clauses, mm in TMDB_QUERIES:
        v, _ = composed(arrs[field], clauses, mm)
        ids, bits = top10(v)
        out["tmdb"].append({"field": field, "clauses": clauses, "mm": mm, "top_ids": ids, "top_bits": bits,
                            "n_ranked": int(np.count_nonzero(v > 0))})
    path = os.path.join(HERE, "bool_scenarios.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print({k: len(v) for k, v in out.items()}, os.path.getsize(path))


if __name__ == "__main__":
    main()
