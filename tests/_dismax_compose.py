"""The composition of boolean queries holding DisMax clauses (tests/golden/make_golden_dismax.py), shared by the CPU
and GPU tests.  A DisMax is one clause: v_j = float32(w_j) * score(member j), d = m + (t - m) * tie with m the
elementwise max and t the left-folded sum of the v_j, matched where any member scores > 0.  Around it, the Bool
composition of tests/_bool_occur_compose.py: s = sum over must + should of weight * score (a DisMax adds d with
weight 1), ranked where s > 0, at least mm should clauses match, every must and filter clause matches and no
must_not clause does.  A top-level DisMax is Bool(should=[it])."""
import numpy as np


def parts(q):
    """(must, must_w, should, should_w, filter, must_not, mm) of an Or / And / Bool / top-level DisMax."""
    from searcharray_b200 import Bool, DisMax
    if isinstance(q, DisMax):
        return [], [], [q], [np.float32(1.0)], [], [], 1
    if isinstance(q, Bool):
        return q.must, q.must_weights, q.should, q.should_weights, q.filter, q.must_not, q.mm
    return [], [], q.clauses, q.weights, [], [], q.mm


def compose_dismax(score, q):
    """score(clause) -> float32[N] for a term / phrase / Field.  The ranked dense vector: s where the doc ranks."""
    from searcharray_b200 import DisMax
    must, must_w, should, should_w, filt, must_not, mm = parts(q)
    cache = {}

    def sc(c):
        key = repr(c)
        if key not in cache:
            cache[key] = np.asarray(score(c), dtype=np.float32)
        return cache[key]

    def value(c):
        """(score, match) of a clause."""
        if not isinstance(c, DisMax):
            return sc(c), sc(c) > 0
        vs = [np.float32(w) * sc(m) for m, w in zip(c.clauses, c.weights)]
        mx = np.maximum.reduce(vs)
        t = vs[0]
        for v in vs[1:]:
            t = t + v
        return mx + (t - mx) * np.float32(c.tie), np.any([sc(m) > 0 for m in c.clauses], axis=0)

    scoring, weights = must + should, list(must_w) + list(should_w)
    s = np.float32(weights[0]) * value(scoring[0])[0]
    for c, w in zip(scoring[1:], weights[1:]):
        s = s + np.float32(w) * value(c)[0]
    hits = np.sum([value(c)[1] for c in should], axis=0) if should else np.zeros(len(s), dtype=np.int64)
    ok = hits >= mm
    for c in must + filt:
        ok &= value(c)[1]
    for c in must_not:
        ok &= ~value(c)[1]
    return np.where(ok & (s > 0), s, np.float32(0)).astype(np.float32)


def query_of(rec):
    """A golden record (make_golden_dismax.py) as the Or / Bool / DisMax it describes: Field leaves, or plain ones
    for a single-field (search_topk) record."""
    from searcharray_b200 import Bool, Boost, DisMax, Field, Or

    def leaf(c):
        x = c["c"] if c["f"] is None else Field(c["f"], c["c"])
        return Boost(x, c["w"]) if c["w"] != 1.0 else x

    def clause(c):
        return DisMax([leaf(m) for m in c["dismax"]], tie=c["tie"]) if "dismax" in c else leaf(c)

    def cs(key):
        return [clause(c) for c in rec[key]]
    if rec["kind"] == "dismax":
        return clause(rec["should"][0])
    if rec["kind"] == "or":
        return Or(cs("should"), mm=rec["mm_spec"])
    return Bool(must=cs("must"), should=cs("should"), filter=cs("filter"), must_not=cs("must_not"),
                mm=rec["mm_spec"])


def record_groups(recs):
    """The records grouped by (single field, slop, per-field similarity): the arguments one call shares."""
    groups = {}
    for r in recs:
        key = (r["field"] or "", r["slop"], tuple(sorted((f, tuple(kb)) for f, kb in r["sim"].items())))
        groups.setdefault(key, []).append(r)
    return groups
