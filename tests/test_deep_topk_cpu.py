"""CPU: the k range of the batched top-k (1 <= k <= 1,024), refused on the host before any device work, and the
Python mirror of SA_TOPK_DEEP_MAX."""
import os
import re

import numpy as np
import pytest

from searcharray_b200.query import TOPK_MAX, check_k

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_mirrors_the_c_header():
    with open(os.path.join(ROOT, "include", "searcharray_b200.h")) as f:
        m = re.search(r"#define SA_TOPK_DEEP_MAX (\d+)", f.read())
    assert m and int(m.group(1)) == TOPK_MAX == 1024


@pytest.mark.parametrize("k", [1, 10, 32, 33, 1000, 1024, np.int64(100)])
def test_accepted(k):
    assert check_k(k) == int(k)


@pytest.mark.parametrize("k", [0, -1, 1025, 4096, 10.0, True, "10"])
def test_refused(k):
    with pytest.raises(ValueError, match=r"k must be in \[1, 1024\]"):
        check_k(k)


def test_fields_topk_refuses_before_device_work():
    import pandas as pd
    from searcharray_b200 import fields_topk
    # an empty frame with no SearchArray column: the k check comes first, so nothing else is looked at
    for k in (0, 1025):
        with pytest.raises(ValueError, match=r"\[1, 1024\]"):
            fields_topk(pd.DataFrame(), ["x"], k=k)
