"""CPU: the phrase phases of the largest edismax query the device path admits (solr._Plan.device_ok) fit what
sa_multi_phrases and sa_multi_add_phase accept (sa_multi.cuh, mirrored in searcharray_b200.query), so that device_ok
and the C checks cannot drift apart again: pf2 on 8 fields of 9 tokens is 72 add_phase entries, once refused."""
import os
import re

import pandas as pd
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def c_define(path, name):
    text = open(os.path.join(ROOT, path)).read()
    return re.search(rf"^#define {name} (.+?)(?:\s*//.*)?$", text, re.M).group(1).strip()


def test_mirrored_limits_match_the_headers():
    from searcharray_b200 import query
    assert int(c_define("include/searcharray_b200.h", "SA_MAX_PHRASE_TERMS")) == query.SA_MAX_PHRASE_TERMS
    assert int(c_define("searcharray_b200/csrc/sa_multi.cuh", "ED_MAX_FIELDS")) == query.ED_MAX_FIELDS
    assert int(c_define("searcharray_b200/csrc/sa_multi.cuh", "ED_MAX_ROWS")) == query.ED_MAX_ROWS
    assert c_define("searcharray_b200/csrc/sa_multi.cuh", "ED_MAX_PHASE_ENTRIES") == "(ED_MAX_FIELDS * SA_MAX_PHRASE_TERMS)"
    assert query.ED_MAX_PHASE_ENTRIES == query.ED_MAX_FIELDS * query.SA_MAX_PHRASE_TERMS


def make_plan(n_fields, n_tokens, boost="^2.5"):
    from searcharray_b200 import SearchArray
    from searcharray_b200.solr import _Plan, default_bm25
    words = [f"w{i}" for i in range(n_tokens)]
    docs = [" ".join(words), " ".join(reversed(words)), "w0 w1"]
    names = [f"f{i}" for i in range(n_fields)]
    frame = pd.DataFrame({f: SearchArray.index(docs) for f in names})
    fields = [f + boost if i % 2 else f for i, f in enumerate(names)]
    return _Plan(frame, " ".join(words), fields, None, fields, fields, fields, 0.3, "OR", default_bm25)


@pytest.mark.parametrize("n_fields,n_tokens", [(8, 16), (8, 9), (1, 16), (8, 2), (3, 3), (5, 16)])
def test_worst_phase_shapes_fit_the_device_limits(n_fields, n_tokens):
    from searcharray_b200.query import ED_MAX_PHASE_ENTRIES, ED_MAX_ROWS
    plan = make_plan(n_fields, n_tokens)
    assert plan.device_ok()
    rows = plan.phrase_rows()
    assert set(rows) == set(plan.names)
    for f, r in rows.items():
        # pf: 1, pf2: T - 1, pf3: T - 2 phrases, each one row of the field's sa_multi_phrases launch
        assert len(r) == 1 + (n_tokens - 1) + max(n_tokens - 2, 0)
        assert len(r) <= ED_MAX_ROWS, (f, len(r))
    entries = dict(plan.phase_entries())
    assert [len(entries[p]) for p in ("pf", "pf2", "pf3")] == \
        [n_fields, n_fields * n_tokens, n_fields * max(n_tokens - 2, 0)]
    for name, e in entries.items():
        assert len(e) <= ED_MAX_PHASE_ENTRIES, (name, len(e))
        for f, row, boost in e:                          # every entry names a row its field computes
            assert 0 <= row < len(rows[f])


def test_pf2_repeats_its_last_bigram_and_rows_follow_phase_order():
    plan = make_plan(2, 4, boost="^3")
    rows = plan.phrase_rows()
    assert rows["f0"] == [("pf", 0), ("pf2", 0), ("pf2", 1), ("pf2", 2), ("pf3", 0), ("pf3", 1)]
    entries = dict(plan.phase_entries())
    assert entries["pf2"] == [("f0", 1, None), ("f0", 2, None), ("f0", 3, None), ("f0", 3, None),
                              ("f1", 1, 3.0), ("f1", 2, 3.0), ("f1", 3, 3.0), ("f1", 3, 3.0)]
    assert entries["pf"] == [("f0", 0, None), ("f1", 0, 3.0)]
    assert entries["pf3"] == [("f0", 4, None), ("f0", 5, None), ("f1", 4, 3.0), ("f1", 5, 3.0)]


def test_device_ok_stops_at_the_limits():
    """One field or one token past the worst shape leaves the device path (composed .score calls instead)."""
    from searcharray_b200.query import ED_MAX_FIELDS, SA_MAX_PHRASE_TERMS
    assert not make_plan(ED_MAX_FIELDS + 1, 2).device_ok()
    assert not make_plan(2, SA_MAX_PHRASE_TERMS + 1).device_ok()
    assert make_plan(ED_MAX_FIELDS, SA_MAX_PHRASE_TERMS).device_ok()
