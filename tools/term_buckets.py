"""Times the batched term path per df bucket, optionally under several settings of the term kernel's tuning knobs
(environment variables read per launch):
    python tools/term_buckets.py [n_docs] [buckets, e.g. 2,3] [queries] [KEY=v1,v2,... ...]
e.g. python tools/term_buckets.py 10000000 1,2,3 128 SA_TERM_QUAD_MIN_RECS=160,512 SA_STAGED_NORM_MIN_RECS=384,768
The value `default` leaves a variable unset (the compiled-in default)."""
import ctypes, itertools, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from searcharray_b200 import _lib, synth
from searcharray_b200.postings import DeviceIndex
from searcharray_b200.similarity import compute_idf

n_docs = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
only = [int(x) for x in sys.argv[2].split(',')] if len(sys.argv) > 2 and sys.argv[2] else None     # 9 = the bench's mix
Q, k = (int(sys.argv[3]) if len(sys.argv) > 3 else 128), 10
knobs = [(a.split('=')[0], a.split('=')[1].split(',')) for a in sys.argv[4:]]
spec = synth.SynthSpec(n_docs, n_phrases=8, n_hard=2, n_bigrams=2)
t0 = time.time()
host, lo, hi = synth.generate_shard(spec)
avgdl = float(synth.global_avg_doc_length(spec))
L = _lib.lib()
dev = DeviceIndex(host, 0, 0)
h = dev.handle
print(f'generated + uploaded in {time.time() - t0:.1f}s', flush=True)
settings = list(itertools.product(*[[(name, v) for v in vals] for name, vals in knobs])) or [()]
for setting in settings:
    for name, v in setting:
        if v == 'default':
            os.environ.pop(name, None)
        else:
            os.environ[name] = v
    print('== ' + (' '.join(f'{n}={v}' for n, v in setting) or 'defaults'), flush=True)
    for b, p in enumerate(synth.DF_BUCKETS):
        if only is not None and b not in only:
            continue
        names = spec.bucket_terms[b]
        tids = np.asarray([spec.term_index[names[j % len(names)]] for j in range(Q)], dtype=np.uint32)
        df = host.term_lengths[tids]
        idf = np.asarray([compute_idf(n_docs, np.asarray([max(1, int(x))])) for x in df], dtype=np.float32).ravel()
        starts = np.arange(Q + 1, dtype=np.uint32)
        _lib.check(L.sa_batch_upload(h, _lib.p_u32(tids), _lib.p_u32(starts), _lib.p_f32(idf), Q, 0, avgdl, 1.2, 0.75, k))
        for _ in range(3):
            _lib.check(L.sa_batch_execute(h))
        ms = ctypes.c_double(0)
        _lib.check(L.sa_timer_start(h))
        for _ in range(8):
            _lib.check(L.sa_batch_execute(h))
        _lib.check(L.sa_timer_stop(h, ctypes.byref(ms)))
        docs = np.empty((Q, k), dtype=np.uint32); scores = np.empty((Q, k), dtype=np.float32); n_over = ctypes.c_uint32(0)
        _lib.check(L.sa_batch_download(h, _lib.p_u32(docs), _lib.p_f32(scores), ctypes.byref(n_over)))
        W = float(np.mean(host.term_lengths[tids]))
        per_q_us = ms.value * 1e3 / (8 * Q)
        print(f"  df/N={p:7.0e}  W={W:10.0f}  {per_q_us:7.2f} us/query  reruns {n_over.value}", flush=True)
    if only is None or 9 in only:
        names = synth.stratified_term_queries(spec, 1024)
        tids = np.asarray([spec.term_index[nm] for nm in names], dtype=np.uint32)
        idf = np.asarray([compute_idf(n_docs, np.asarray([max(1, int(x))])) for x in host.term_lengths[tids]], dtype=np.float32).ravel()
        starts = np.arange(len(tids) + 1, dtype=np.uint32)
        _lib.check(L.sa_batch_upload(h, _lib.p_u32(tids), _lib.p_u32(starts), _lib.p_f32(idf), len(tids), 0, avgdl, 1.2, 0.75, k))
        for _ in range(3):
            _lib.check(L.sa_batch_execute(h))
        ms = ctypes.c_double(0)
        _lib.check(L.sa_timer_start(h))
        for _ in range(10):
            _lib.check(L.sa_batch_execute(h))
        _lib.check(L.sa_timer_stop(h, ctypes.byref(ms)))
        print(f"  mix of 1024 distinct terms: {ms.value / 10:7.3f} ms/step = {1024 * 10 / ms.value * 1e3:9.0f} q/s", flush=True)
