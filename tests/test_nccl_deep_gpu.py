"""World-size-2 NCCL run of the sharded scoring path at deep k (k = 100 and 1,024): each shard's deep collector, one
ncclAllGather of the per-shard top k and the device merge, against the CPU oracle on the full corpus.  Skips with
fewer than 2 GPUs.  The merge kernels themselves, for 1 to 8 ranks and k up to 1,024, run on one GPU in
test_deep_topk_gpu.py (sa_topk_merge)."""
import ctypes
import os
import subprocess
import sys

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu


def gpu_count():
    from searcharray_b200 import _lib
    n = ctypes.c_int(0)
    _lib.check(_lib.lib().sa_device_count(ctypes.byref(n)))
    return n.value


def test_two_gpu_allgather_deep_topk_matches_oracle():
    if gpu_count() < 2:
        pytest.skip("needs 2 GPUs")
    key = f"/tmp/sa_b200_deep_uid_{os.getpid()}.bin"
    if os.path.exists(key):
        os.remove(key)
    env = dict(os.environ)
    env.pop("NCCL_DEBUG", None)
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_nccl_deep_worker.py"), str(r), "2", key],
                              env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = []
    try:
        for p in procs:
            out, _ = p.communicate(timeout=900)
            outs.append(out)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        if os.path.exists(key):
            os.remove(key)
    assert all(p.returncode == 0 for p in procs), "\n".join(o[-2000:] for o in outs)
    assert "NCCL_DEEP_OK 2" in outs[0], outs[0][-2000:]
