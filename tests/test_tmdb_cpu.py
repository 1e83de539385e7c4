"""BASELINE configs[0]: the TMDB fixture (27,846 real documents) -- the host indexer and the CPU
oracle against what the REAL reference produced on it (tests/golden/tmdb.json: digests, counts and
top-10 lists; made by tests/golden/make_golden_tmdb.py).  The corpus enters as the stored index of both
fields (tests/golden/tmdb_index.npz, the same file the GPU tests upload), which is first checked against
the reference's own index digest.  The indexer is checked by re-indexing the token streams that index
holds (every token of every document at its position, joined by single spaces)."""
import hashlib
import json
import os

import numpy as np
import pytest

from _tmdb_index import load_field
from conftest import GOLDEN

G = json.load(open(os.path.join(GOLDEN, "tmdb.json")))


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def index_digest(host):
    """The reference's canonical digest (make_golden_tmdb.index_digest) of a HostIndex."""
    h = hashlib.sha256()
    t2i = host.term_dict.term_to_ids
    for t in sorted(t2i.keys()):
        h.update(t.encode("utf-8"))
        h.update(np.ascontiguousarray(host.term_words(t2i[t]), dtype=np.uint64).tobytes())
    return {"n_terms": host.n_terms, "n_words": len(host.words), "sha256": h.hexdigest(),
            "doc_lens_sha256": sha(host.doc_lens.astype(np.float32)), "avg_doc_length": float(host.avg_doc_length)}


def token_streams(host):
    """Each document's tokens in position order, decoded from the roaringish words
    (doc id << 36 | position block << 18 | one bit per position in the block)."""
    from searcharray_b200.roaringish import LSB_BITS
    words = host.words.astype(np.uint64)
    order = np.argsort(host.term_offsets, kind="stable")
    term_of_word = np.repeat(order, host.term_lengths[order].astype(np.int64))
    assert len(term_of_word) == len(words)
    doc = (words >> np.uint64(36)).astype(np.int64)
    base = ((words >> np.uint64(LSB_BITS)) & np.uint64(0x3FFFF)).astype(np.int64) * LSB_BITS
    d, p, t = [], [], []
    for bit in range(LSB_BITS):
        on = ((words >> np.uint64(bit)) & np.uint64(1)).astype(bool)
        d.append(doc[on]); p.append(base[on] + bit); t.append(term_of_word[on])
    d, p, t = np.concatenate(d), np.concatenate(p), np.concatenate(t)
    srt = np.lexsort((p, d))
    d, p, t = d[srt], p[srt], t[srt]
    names = [host.term_dict.get_term(i) for i in range(host.n_terms)]
    counts = np.bincount(d, minlength=host.n_docs)
    assert np.array_equal(counts, host.doc_lens.astype(np.int64))
    starts = np.concatenate(([0], np.cumsum(counts)))
    assert np.array_equal(p, np.arange(len(p)) - np.repeat(starts[:-1], counts))   # positions 0..len-1
    return [" ".join(names[i] for i in t[starts[k]:starts[k + 1]]) for k in range(host.n_docs)]


@pytest.fixture(scope="module")
def fields():
    from oracle import search as osearch, solr as osolr
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    out = {}
    for name in ("title_tokens", "overview_tokens"):
        host = load_field(z, name)
        assert index_digest(host) == G["fields"][name]["index"], name      # the reference's index, word for word
        assert host.n_docs == G["n_docs"]
        idx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                  avg_doc_length=host.avg_doc_length)
        out[name] = (host, osolr.OracleField(idx, host.term_dict.term_to_ids))
    return out


def check_vec(got, rec, what):
    got = np.asarray(got)
    assert str(got.dtype) == rec["dtype"], what
    assert int(np.count_nonzero(got)) == rec["nonzero"], what
    order = np.lexsort((np.arange(len(got)), -got.astype(np.float64)))[:10]
    order = order[got[order] > 0]
    assert [int(i) for i in order] == rec["top_ids"], what
    assert sha(got) == rec["sha256"], what            # the whole vector, bit for bit


@pytest.mark.parametrize("field", ["title_tokens", "overview_tokens"])
def test_host_indexer_matches_reference_index(fields, field):
    """searcharray_b200.indexing.build_index on the corpus's token streams == the reference's index, word for word."""
    from searcharray_b200.indexing import build_index
    stored, _ = fields[field]
    host = build_index(token_streams(stored), str.split)
    assert index_digest(host) == G["fields"][field]["index"]
    assert host.n_docs == G["n_docs"]


@pytest.mark.parametrize("field", ["title_tokens", "overview_tokens"])
def test_oracle_terms_and_phrases_on_tmdb(fields, field):
    from oracle import ops as oops
    _, of = fields[field]
    rec = G["fields"][field]
    for term, r in rec["terms"].items():
        tid = of.term_to_id.get(term)
        assert int(of.index.docfreq(tid)) == r["df"], term
        check_vec(of.index.termfreqs(tid), r["tf"], (field, term, "tf"))
        check_vec(of.index.score(tid), r["score"], (field, term, "score"))
    for r in rec["phrases"]:
        ids = of.ids(r["phrase"])
        check_vec(of.index.termfreqs(ids), r["tf"], (field, r["phrase"], "tf"))
        check_vec(of.index.score(ids), r["score"], (field, r["phrase"], "score"))
    for r in rec["slop"]:
        got = of.index.termfreqs(of.ids(r["phrase"]), slop=r["slop"])
        if not oops.last_span_undefined:
            check_vec(got, r["tf"], (field, r["phrase"], r["slop"]))


def test_oracle_edismax_on_tmdb(fields):
    """reference test/test_tmdb.py:230-241: qf + pf + pf2 + pf3 over title and overview, mm=2, tie=0.3."""
    from oracle import solr as osolr
    ofields = {name: f for name, (_, f) in fields.items()}
    for r in G["edismax"]:
        got = osolr.edismax(ofields, r["q"], **G["edismax_kwargs"])
        check_vec(got, r["scores"], r["q"])
