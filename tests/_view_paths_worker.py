"""Worker for tests/test_view_paths_gpu.py: the document-frequency checks and term queries on views in a process
started with SA_NO_TF_TABLE=1, which the library reads once per process, so that every list takes the words branch of
docfreq_rows_kernel (jobs of 4,096 words) and the term scan's words path.  Prints OK when every check passes."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_view_paths_gpu as paths  # noqa: E402


def main():
    assert os.environ.get("SA_NO_TF_TABLE") == "1"
    ctx = paths.Ctx()
    paths.check_docfreqs(ctx, "words")
    terms = ["r0", "r1", "edge", "straddle", "f5000", "s0", "zzz"]
    for kind, vname in ((paths.BM25, "mask"), (paths.BM25, "repeats"), (paths.LEGACY, "unsliced"),
                        (paths.CLASSIC, "stepped")):
        paths.check_kind_view(ctx, kind, vname, queries=terms, slops=(0,), ks=(1, 17, 32))
    print("OK")


if __name__ == "__main__":
    main()
