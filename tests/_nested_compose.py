"""The composition of boolean queries holding nested queries (tests/golden/make_golden_nested.py), shared by the CPU and
GPU tests and tools/nested_topk_bench.py.  It is compose_dismax's (tests/_dismax_compose.py) with one more kind of
clause: a nested Or / And / Bool N scores r_N = compose(N), the dense vector N ranks as a query of its own, and
matches where r_N > 0.  Around it nothing changes: must / should add float32(w) * r_N, it counts once towards its
parent's mm, and under filter / must_not it plays a leaf's role."""
import numpy as np

from _dismax_compose import parts


def compose_nested(score, q, _cache=None):
    """score(clause) -> float32[N] for a term / phrase / Field.  The ranked dense vector of q: s where the doc ranks,
    +0 elsewhere."""
    from searcharray_b200 import Bool, DisMax, Or
    cache = {} if _cache is None else _cache
    must, must_w, should, should_w, filt, must_not, mm = parts(q)

    def sc(c):
        key = repr(c)
        if key not in cache:
            cache[key] = np.asarray(score(c), dtype=np.float32)
        return cache[key]

    def value(c):
        """(score, match) of a clause."""
        if isinstance(c, (Or, Bool)):
            r = compose_nested(score, c, cache)
            return r, r > 0
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
    """A golden record (make_golden_nested.py) or one of its nested nodes as the Or / Bool it describes: a leaf is
    {"f", "c", "w"} (Field leaves, or plain ones for a single-field record), a DisMax {"dismax": [leaves], "tie"}, a
    nested query {"node": record, "w"}."""
    from searcharray_b200 import Bool, Boost, DisMax, Field, Or

    def boost(x, w):
        return Boost(x, w) if w != 1.0 else x

    def clause(c):
        if "node" in c:
            return boost(query_of(c["node"]), c["w"])
        if "dismax" in c:
            return DisMax([clause(m) for m in c["dismax"]], tie=c["tie"])
        return boost(c["c"] if c["f"] is None else Field(c["f"], c["c"]), c["w"])

    def cs(key):
        return [clause(c) for c in rec.get(key, [])]
    if rec["kind"] == "or":
        return Or(cs("should"), mm=rec["mm_spec"])
    return Bool(must=cs("must"), should=cs("should"), filter=cs("filter"), must_not=cs("must_not"),
                mm=rec["mm_spec"])
