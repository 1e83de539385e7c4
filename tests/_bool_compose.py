"""The reference's composition of a boolean query (test/test_search.py:126-226), shared by the CPU and GPU boolean
tests: per doc s = score(c0) + score(c1) + ... folded left in float32, ranked where s > 0 and at least mm clauses
score > 0, top k by (score desc, id asc)."""
import numpy as np

NO_DOC = 0xFFFFFFFF


def compose(score, clauses, mm):
    """score(clause) -> float32[N].  Returns (s where the doc ranks else 0, the mm mask)."""
    scores = [np.asarray(score(c), dtype=np.float32) for c in clauses]
    s = scores[0]
    for v in scores[1:]:
        s = s + v
    ok = np.sum(np.array(scores) > 0, axis=0) >= mm
    return np.where(ok & (s > 0), s, np.float32(0)).astype(np.float32), ok


def topk(dense, k, doc_base=0):
    """(ids uint32[k], scores float32[k]) of the k best scores > 0 by (score desc, id asc); empty NO_DOC / 0."""
    dense = np.asarray(dense, dtype=np.float32)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=np.float32)
    docs[:len(order)] = order + doc_base
    scores[:len(order)] = dense[order]
    return docs, scores


def oracle_score(oidx, term_dict, k1=1.2, b=0.75, slop=0):
    """score(clause) over an oracle.search.OracleIndex; tokens missing from term_dict score zero."""
    def tid(t):
        return term_dict.term_to_ids.get(t)

    def score(c):
        ids = tid(c) if isinstance(c, str) else [tid(t) for t in c]
        return oidx.score(ids, k1=k1, b=b, slop=slop)
    return score


def expand(rec):
    """A period-compressed list of the fixture ({"base": [...], "times": n}) back to the list."""
    return list(rec["base"]) * rec["times"]
