"""The image post-processing drop-in header: tests/cpp/image_dropin_example.cpp builds with plain g++ against
include/ouster/core/image_processing.h and runs on the GPU; every result equals the oracle's (oracle/orc_image.c).
The new ABI structs compile as C99."""
import os
import subprocess

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import image as oi

ROOT = graft.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "image_dropin_example.cpp")
LIB_DIR = os.path.join(ROOT, "ouster-sdk_b200", "lib")


def build_example(out_dir):
    graft.build()
    exe = os.path.join(str(out_dir), "image_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"),
                           SRC, "-L", LIB_DIR, "-louster_b200", f"-Wl,-rpath,{LIB_DIR}", "-o", exe])
    return exe


def test_image_structs_are_plain_c99(tmp_path):
    graft.build()
    src = tmp_path / "image.c"
    src.write_text('#include "ouster_b200.h"\n'
                   "int main(void) { ob_image_params p = {0}; ob_image_state s = {0}; ob_image_proc* h = 0;\n"
                   "  (void)p; (void)s; (void)h;\n"
                   "  return ob_abi_sizeof(\"ob_image_params\") == sizeof(p) &&\n"
                   "         ob_abi_sizeof(\"ob_image_state\") == sizeof(s) && OB_IMAGE_RGB_F16 == 2 &&\n"
                   "         OB_IMAGE_LOCAL_TONE_MAP == 2 ? 0 : 1; }\n")
    exe = tmp_path / "image"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I",
                           os.path.join(ROOT, "include"), str(src), "-L", LIB_DIR, "-louster_b200",
                           f"-Wl,-rpath,{LIB_DIR}", "-o", str(exe)])
    assert subprocess.run([str(exe)]).returncode == 0


def test_image_dropin_example_compiles(tmp_path):
    assert os.path.exists(build_example(tmp_path))


@pytest.mark.gpu
def test_image_dropin_example_runs_on_gpu(tmp_path):
    h, w, frames = 32, 256, 5
    r = np.random.default_rng(11)
    mono = (r.uniform(1, 50, (frames, h, w)) + np.linspace(0, 5, h)[:, None]).astype(np.float32)
    mono[r.random(mono.shape) < 0.2] = 0
    rgb = r.uniform(0, 20, (frames, h, w, 3)).astype(np.float32)
    half = r.uniform(0, 1.5, (frames, h, w, 3)).astype(np.float16)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(mono.tobytes() + rgb.tobytes() + half.tobytes())
    out_bin = tmp_path / "out.bin"
    out = subprocess.run([build_example(tmp_path), str(h), str(w), str(frames), str(inp), str(out_bin)],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "IMAGE DROPIN OK" in out.stdout
    raw = out_bin.read_bytes()
    n = frames * h * w
    sizes = [(np.float32, n), (np.float64, n), (np.float32, 3 * n), (np.float32, 3 * n), (np.float32, 3 * n)]
    got, at = [], 0
    for dt, k in sizes:
        got.append(np.frombuffer(raw, dt, k, at))
        at += k * np.dtype(dt).itemsize
    assert at == len(raw)
    ae, buc, ae_rgb, ae_half, ltm = (oi.AutoExposure(), oi.BeamUniformityCorrector(), oi.AutoExposure(),
                                     oi.AutoExposure(), oi.LocalToneMapper())
    want = [[] for _ in range(5)]
    for f in range(frames):
        us = f != 2
        a, d, c = mono[f].copy(), mono[f].astype(np.float64), rgb[f].copy()
        ae.update(a, us)
        buc.update(d, us)
        ae_rgb.update(c, us)
        for lst, v in zip(want, (a, d, c, ae_half.update(half[f], us), ltm.update(half[f], us))):
            lst.append(v.reshape(-1))
    for k in range(5):
        assert np.array_equal(got[k], np.concatenate(want[k]), equal_nan=True), k
