"""The composition of a Bool / boosted Or query (tests/golden/make_golden_bool_occur.py), shared by the CPU and GPU
tests: s = w0 * score(c0) + w1 * score(c1) + ... over must + should (float32, each product rounded, folded left),
ranked where s > 0, at least mm should clauses score > 0, every must and filter clause scores > 0 and no must_not
clause does."""
import numpy as np


def parts(q):
    """(must, must_w, should, should_w, filter, must_not, mm) of an Or / And / Bool."""
    from searcharray_b200 import Bool
    if isinstance(q, Bool):
        return q.must, q.must_weights, q.should, q.should_weights, q.filter, q.must_not, q.mm
    return [], [], q.clauses, q.weights, [], [], q.mm


def compose_occur(score, q):
    """score(clause) -> float32[N].  The ranked dense vector: s where the doc ranks, else 0."""
    must, must_w, should, should_w, filt, must_not, mm = parts(q)
    cache = {}

    def sc(c):
        key = repr(c)
        if key not in cache:
            cache[key] = np.asarray(score(c), dtype=np.float32)
        return cache[key]
    scoring, weights = must + should, list(must_w) + list(should_w)
    s = np.float32(weights[0]) * sc(scoring[0])
    for c, w in zip(scoring[1:], weights[1:]):
        s = s + np.float32(w) * sc(c)
    hits = np.sum([sc(c) > 0 for c in should], axis=0) if should else np.zeros(len(s), dtype=np.int64)
    ok = hits >= mm
    for c in must + filt:
        ok &= sc(c) > 0
    for c in must_not:
        ok &= ~(sc(c) > 0)
    return np.where(ok & (s > 0), s, np.float32(0)).astype(np.float32)


def query_of(rec):
    """A golden record (make_golden_bool_occur.py) as the Or / Bool it describes."""
    from searcharray_b200 import Bool, Boost, Or

    def boosted(cs, ws):
        return [Boost(c, w) if w != 1.0 else c for c, w in zip(cs, ws)]
    if rec["kind"] == "or":
        return Or(boosted(rec["should"], rec["should_w"]), mm=rec["mm"])
    return Bool(must=boosted(rec["must"], rec["must_w"]), should=boosted(rec["should"], rec["should_w"]),
                filter=rec["filter"], must_not=rec["must_not"], mm=rec["mm"])
