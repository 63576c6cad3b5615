"""Several JOIN clauses per query and expression join keys in the QL evaluator (host/tests/multi_join_ut.cpp).

The C++ test holds hand-written queries over spelled-out rows, a randomized check against a CPU model of the chain
(nested-loop joins in lexicographic order, NULL = NULL, doubles by bit pattern) and an equivalence check of two clauses
against two single-clause queries.  Here it is built, refused without a device, and run on the GPU.
"""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "multi_join_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "multi_join_ut")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 100 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_gpu_host_adapter_join_chain():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "multi_join_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "multi_join_ut")], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-4000:]
    assert "multi_join_ut: 0 failure(s)" in r.stdout
