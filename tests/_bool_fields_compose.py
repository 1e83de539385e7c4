"""The composition of a boolean query over several fields (tests/golden/make_golden_bool_fields.py), shared by the CPU
and GPU tests: compose_occur (tests/_bool_occur_compose.py) with score(Field(f, c)) = the field's own score(c)."""


def field_scorer(scorers):
    """scorers: field -> score(clause).  The score(Field) compose_occur takes."""
    return lambda c: scorers[c.field](c.clause)


def query_of(rec):
    """A golden record (make_golden_bool_fields.py) as the Or / Bool of Field clauses it describes."""
    from searcharray_b200 import Bool, Boost, Field, Or

    def fc(c):
        return Field(c["f"], c["c"])

    def boosted(cs, ws):
        return [Boost(fc(c), w) if w != 1.0 else fc(c) for c, w in zip(cs, ws)]
    if rec["kind"] == "or":
        return Or(boosted(rec["should"], rec["should_w"]), mm=rec["mm_spec"])
    return Bool(must=boosted(rec["must"], rec["must_w"]), should=boosted(rec["should"], rec["should_w"]),
                filter=[fc(c) for c in rec["filter"]], must_not=[fc(c) for c in rec["must_not"]], mm=rec["mm_spec"])


def record_groups(recs):
    """The records grouped by (slop, per-field similarity), the arguments one fields_topk call shares."""
    groups = {}
    for r in recs:
        key = (r["slop"], tuple(sorted((f, tuple(kb)) for f, kb in r["sim"].items())))
        groups.setdefault(key, []).append(r)
    return groups
