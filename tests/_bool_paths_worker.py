"""Worker for tests/test_bool_paths_gpu.py: the records-term and tf = 2^18 checks in a process started with
SA_NO_TF_TABLE=1, which the library reads once per process, so that every long list takes the words path over its tile
directory.  Prints OK when every check passes."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_bool_paths_gpu as paths  # noqa: E402


def main():
    assert os.environ.get("SA_NO_TF_TABLE") == "1"
    paths.check_records_paths(paths.Ctx(), "no tf table")
    print("OK")


if __name__ == "__main__":
    main()
