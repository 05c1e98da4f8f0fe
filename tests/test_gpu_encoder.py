"""Encoder-level proof of the drop-in boundary (SURVEY 8c "End-to-end oracle", BASELINE configs[0]): the UNMODIFIED reference
encoder + CLI, linked with setupCudaPrimitives() at the primitives.cpp:264 position (oracle/encoder_cuda_hook.cpp, selector
X265_PRIMITIVES=cuda), must produce the same bitstream as the C table (--no-asm) on the synthetic CIF clip; and a CUDA
failure inside a per-call primitive must surface as an error flag, never as a killed process."""
import ctypes as C
import hashlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from common import ROOT
from frame_helpers import gen_luma, gen_chroma

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "oracle", "_ref", "x265_ref_cuda")


def write_cif(path, frames):
    W, H = 352, 288
    with open(path, "wb") as f:
        for n in range(frames):
            f.write(gen_luma(W, H, n, s1=17.0, s2=11.0).tobytes())
            f.write(gen_chroma(W, H, n, 1).tobytes())
            f.write(gen_chroma(W, H, n, 2).tobytes())


@pytest.mark.timeout(900)
def test_encoder_bitstream_equals_c_table(tmp_path):
    if not os.path.exists(CLI):
        pytest.skip("oracle/_ref/x265_ref_cuda not built: the encoder is linked from the reference's sources, so it exists only "
                    "where build() had them (make -C oracle -f Makefile.ref encoder_cuda)")
    frames = 3
    yuv = str(tmp_path / "cif.yuv")
    write_cif(yuv, frames)
    md5, logs = {}, {}
    for mode in ("c", "cuda"):
        out = str(tmp_path / ("out_%s.hevc" % mode))
        env = dict(os.environ)
        env.pop("X265_PRIMITIVES", None)
        if mode == "cuda":
            env["X265_PRIMITIVES"] = "cuda"
        cmd = [CLI, "--input", yuv, "--input-res", "352x288", "--fps", "30", "--preset", "ultrafast", "--no-asm", "--pools", "4", "-F", "1",
               "--frames", str(frames), "-o", out]
        r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=850)
        logs[mode] = r.stdout
        assert r.returncode == 0, r.stdout[-2000:]
        md5[mode] = hashlib.md5(open(out, "rb").read()).hexdigest()
        assert os.path.getsize(out) > 1000
    m = re.search(r"per-call primitives executed on the device: (\d+), error flag: (\d+)", logs["cuda"])
    assert m, logs["cuda"][-2000:]
    assert int(m.group(1)) > 1000 and int(m.group(2)) == 0, m.group(0)
    assert "EncoderPrimitives table = CUDA" in logs["cuda"] and "table = CUDA" not in logs["c"]
    assert md5["c"] == md5["cuda"], (md5, logs["cuda"][-1500:])


def test_primitive_failure_sets_flag_and_process_survives(tmp_path):
    """Fault injection: the per-call table bound to a device that does not exist.  The primitive returns (zeros), the flag
    x265cu_primitive_error() is latched with a message, and the process keeps running."""
    code = r'''
import ctypes as C, sys
sys.path.insert(0, %r)
import x265_b200
lib = x265_b200.load(need_gpu=False)
assert lib.L.x265cu_primitive_error() == 0
f = lib.primitive(8, "pu.sad", C.c_int, [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t], 1)
assert f is not None
a = (C.c_uint8 * (64 * 64))(*([7] * 4096)); b = (C.c_uint8 * (64 * 64))(*([9] * 4096))
v = f(C.addressof(a), 64, C.addressof(b), 64)
print("returned", v, "flag", lib.L.x265cu_primitive_error(), lib.L.x265cu_primitive_error_string().decode())
assert lib.L.x265cu_primitive_error() == 1
lib.L.x265cu_primitive_error_clear()
assert lib.L.x265cu_primitive_error() == 0
print("ALIVE")
''' % ROOT
    env = dict(os.environ, X265CU_DEVICE="99")
    r = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 0 and "ALIVE" in r.stdout, r.stdout[-1500:]
