"""Worker for tests/test_deep_topk_gpu.py: the deep term kernel's words path in a process started with
SA_NO_TF_TABLE=1 and SA_TERM_QUERY_MAJOR=1, which the library reads once per process.  Prints OK when every check
passes."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import pytest  # noqa: E402

import test_deep_topk_gpu as deep  # noqa: E402


def main():
    from searcharray_b200 import SearchArray, bm25_similarity
    arr = SearchArray.index(deep.random_corpus(np.random.default_rng(7), 3 * deep.TILE + 1234, 400))
    env = pytest.MonkeyPatch()
    for setting in ("default", "always", "never"):
        for var in ("SA_STAGED_NORM_MIN_RECS", "SA_STAGED_NORM_MIN_WORDS", "SA_TERM_QUAD_MIN_RECS"):
            env.delenv(var, raising=False)
        for var, val in deep.KNOBS[setting].items():
            env.setenv(var, val)
        dense = deep.oracle_dense(arr, deep.TERMS)
        deep.check_queries(arr, deep.TERMS, dense, what=("words", setting))
        deep.check_prefix(arr, deep.TERMS, what=("words", setting))
    sim = bm25_similarity(k1=1.2, b=1.0)                   # the ALL_DOCS instance
    deep.check_queries(arr, deep.TERMS, [arr.score(q, similarity=sim) for q in deep.TERMS], ks=(33, 1024),
                       what="words exotic", similarity=sim)
    print("OK")


if __name__ == "__main__":
    main()
