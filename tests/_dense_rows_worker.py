"""Worker for tests/test_dense_rows_gpu.py: one batch of every kind on the 2M-doc synthetic corpus, in a process whose
SA_DENSE_PLAIN setting (read once per process) picks where the term batch's rare-term rows live.  Prints one JSON line:
whether those rows were compressible, and a digest of every result."""
import ctypes
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402


def main():
    from searcharray_b200 import SearchArray, _lib, synth
    spec = synth.SynthSpec(2_000_000)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    h = hashlib.sha256()
    names = [nm for bi in range(len(synth.DF_BUCKETS)) for nm in spec.bucket_terms[bi][:40]]
    for q in (names, [nm for bi in (4, 5) for nm in spec.bucket_terms[bi][:5]]):
        docs, scores = arr.search_topk(q, k=10)
        h.update(np.ascontiguousarray(docs).tobytes())
        h.update(np.ascontiguousarray(scores).tobytes())
    m = ctypes.c_int(-1)
    _lib.check(_lib.lib().sa_index_dense_compressible(arr._device().handle, ctypes.byref(m)))
    phrases = [ph["terms"] for ph in spec.phrases[:24]]
    for slop in (0, 2):
        docs, scores = arr.search_topk(phrases, k=10, slop=slop)
        h.update(np.ascontiguousarray(docs).tobytes())
        h.update(np.ascontiguousarray(scores).tobytes())
    mixed = names[::7] + phrases[:6]
    docs, scores = arr.search_topk(mixed, k=10)
    h.update(np.ascontiguousarray(docs).tobytes())
    h.update(np.ascontiguousarray(scores).tobytes())
    for bi in range(len(synth.DF_BUCKETS)):
        h.update(np.ascontiguousarray(arr.score(spec.bucket_terms[bi][0])).tobytes())
    print(json.dumps({"compressible": m.value, "digest": h.hexdigest()}))


if __name__ == "__main__":
    main()
