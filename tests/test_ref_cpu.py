"""The oracle port (oracle/search.py + oracle/sa_oracle.c) against the REAL reference on the seeded synthetic
corpus -- the same index object both arms of bench.py run on.  What the reference returned on it is stored as
whole-vector SHA-256 digests in tests/golden/ref_synth.json (tests/golden/make_golden_ref_outputs.py)."""
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN

G = json.load(open(os.path.join(GOLDEN, "ref_synth.json")))


@pytest.fixture(scope="module")
def corpus():
    from oracle import search as osearch
    from searcharray_b200 import synth
    spec = synth.SynthSpec(300_000, terms_per_bucket=5, n_phrases=16, n_bigrams=4)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=avgdl, corpus_size=host.n_docs, cache=True)
    return spec, host, oidx


def sha(a):
    a = np.asarray(a)
    assert a.dtype == np.float32
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_terms_match_the_reference(corpus):
    spec, host, oidx = corpus
    assert sorted(G["terms"]) == sorted(name for name, _, _ in spec.terms)
    for t, (name, _, _) in enumerate(spec.terms):
        want = G["terms"][name]
        assert int(oidx.docfreq(t)) == want["df"], name
        assert sha(oidx.termfreqs(t)) == want["tf"], name
        assert sha(oidx.score(t, k1=1.2, b=0.75)) == want["score"], name
    assert sha(oidx.score(None)) == G["missing_score"]


def test_phrases_and_slop_match_the_reference(corpus):
    spec, host, oidx = corpus
    n_match = 0
    assert [ph["terms"] for ph in spec.phrases] == [w["terms"] for w in G["phrases"]]
    for ph, want in zip(spec.phrases, G["phrases"]):
        ids = [spec.term_index[t] for t in ph["terms"]]
        got = oidx.termfreqs(ids)
        assert sha(got) == want["tf"], ph
        assert sha(oidx.score(ids, k1=1.2, b=0.75)) == want["score"], ph
        n_match += int(np.count_nonzero(got))
    assert n_match > 0
    from oracle import ops as oops
    for ph, want in zip(spec.phrases[::3], G["slop2"]):
        ids = [spec.term_index[t] for t in ph["terms"]]
        got = oidx.termfreqs(ids, slop=2)
        if not oops.last_span_undefined:
            assert sha(got) == want["tf"], ph
