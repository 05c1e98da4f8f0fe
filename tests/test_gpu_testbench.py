"""GPU parity through the reference's OWN test harness: oracle/_ref/testbench_cuda{8,10} link the
unmodified reference harnesses (source/test/{pixel,mbdst,ipfilter,intrapred}harness.cpp) against the
reference C table and against setupCudaPrimitives() (x265_b200/plugin), and run
testCorrectness(cprim, cudaprim) exactly as source/test/testbench.cpp:155-233 does for the asm table."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("seed", [265, 1])
def test_reference_testbench(depth, seed):
    exe = os.path.join(ROOT, "oracle", "_ref", "testbench_cuda%d" % depth)
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/testbench_cuda%d not built: it links the reference's own harness sources, so it exists only "
                    "where build() had them; test_gpu_table.py compares the same entries with the oracle, and test_oracle_vs_ref.py "
                    "the oracle with the reference's stored results" % depth)
    r = subprocess.run([exe, str(seed)], capture_output=True, text=True, timeout=900)
    tail = (r.stdout[-1500:] + r.stderr[-1500:])
    assert r.returncode == 0, tail
    assert "all reference harnesses passed" in r.stdout, tail
