"""Worker for tests/test_term_paths_gpu.py: the branch matrix of the term scan in a process started with
SA_NO_TF_TABLE=1 and SA_TERM_QUERY_MAJOR=1, which the library reads once per process.  Prints OK when every check
passes."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import pytest  # noqa: E402

import test_term_paths_gpu as paths  # noqa: E402


def main():
    case = paths.Case(*paths.mixed_corpus())
    env = pytest.MonkeyPatch()
    for setting in ("default", "always", "never"):
        paths.set_knobs(env, setting)
        paths.check_mixed(case, f"no tf table, query-major, {setting}")
    print("OK")


if __name__ == "__main__":
    main()
