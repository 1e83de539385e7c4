"""Worker for tests/test_nested_gpu.py: the nested-query role checks in a process started with SA_NO_TF_TABLE=1, which the
library reads once per process, so the long lists of every field take the words path with a tile directory.  Prints
OK when every check passes."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_nested_gpu as dm  # noqa: E402


def main():
    assert os.environ.get("SA_NO_TF_TABLE") == "1"
    synth = dm.Frame()
    dm.check_roles(synth.frame, synth.score(), "no tf table")
    print("OK")


if __name__ == "__main__":
    main()
