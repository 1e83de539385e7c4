"""Boolean queries for SearchArray.search_topk: OR / AND / min-should-match over term and phrase clauses.

Or(clauses, mm) ranks, per doc, s = score(c0) + score(c1) + ... (float32, folded left in clause order) among the docs
where at least mm clauses score > 0 -- the reference's own composition of multi-clause queries
(test/test_search.py:126-226) -- and search_topk returns the top k of it by (score desc, doc asc), computed on the
device (sa_score_batch_topk_bool)."""
from typing import List, Union

import numpy as np

from .solr import parse_min_should_match

SA_BOOL_MAX_CLAUSES = 64          # include/searcharray_b200.h

Clause = Union[str, List[str]]


class Or:
    """A query matching docs where at least `mm` of `clauses` score > 0, scored by the sum of the clauses' scores.

    clauses: a str (a term) or a list[str] (a phrase, matched with search_topk's `slop`); duplicates count twice.
    mm: an int or a Solr min-should-match spec ("2", "-1", "75%", "2<-25%"), clamped to [0, len(clauses)] as
    edismax clamps it (solr.parse_min_should_match)."""

    def __init__(self, clauses, mm=1):
        clauses = list(clauses)
        if not clauses:
            raise ValueError("a boolean query needs at least one clause")
        if len(clauses) > SA_BOOL_MAX_CLAUSES:
            raise ValueError(f"a boolean query has at most {SA_BOOL_MAX_CLAUSES} clauses, not {len(clauses)}")
        out = []
        for c in clauses:
            if isinstance(c, str):
                out.append(c)
            elif isinstance(c, (list, tuple)) and c and all(isinstance(t, str) for t in c):
                out.append(list(c))
            else:
                raise TypeError(f"a clause is a str (term) or a non-empty list of str (phrase), not {c!r}")
        self.clauses = out
        self.mm = parse_min_should_match(len(out), str(mm))

    def __repr__(self):
        return f"{type(self).__name__}({self.clauses!r}, mm={self.mm})"


class And(Or):
    """Every clause must score > 0: Or(clauses, mm=len(clauses))."""

    def __init__(self, clauses):
        clauses = list(clauses)
        super().__init__(clauses, mm=len(clauses))


def flatten(queries):
    """Boolean queries as sa_score_batch_topk_bool takes them: (clause list in query order, query_clause_starts,
    mm), the clause list being search_topk's query form (str or list[str])."""
    clauses, starts, mm = [], [0], []
    for q in queries:
        clauses.extend(q.clauses)
        starts.append(len(clauses))
        mm.append(q.mm)
    return clauses, np.asarray(starts, dtype=np.uint32), np.asarray(mm, dtype=np.uint32)
