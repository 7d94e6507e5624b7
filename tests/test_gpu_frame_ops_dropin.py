"""The frame operations drop-in header: tests/cpp/frame_ops_dropin_example.cpp builds with plain g++ against
include/ouster/core/frame_ops.h and runs on the GPU; every field equals the oracle's (oracle/frame_ops.py) and the
error texts are the reference's."""
import os
import subprocess

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import frame_ops as ofo

ROOT = graft.ROOT
SRC = os.path.join(ROOT, "tests", "cpp", "frame_ops_dropin_example.cpp")
LIB_DIR = os.path.join(ROOT, "ouster-sdk_b200", "lib")


def build_example(out_dir):
    graft.build()
    exe = os.path.join(str(out_dir), "frame_ops_dropin_example")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"),
                           SRC, "-L", LIB_DIR, "-louster_b200", f"-Wl,-rpath,{LIB_DIR}", "-o", exe])
    return exe


def test_frame_ops_dropin_example_compiles(tmp_path):
    assert os.path.exists(build_example(tmp_path))


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(16, 256), (7, 333)])
def test_frame_ops_dropin_example_runs_on_gpu(tmp_path, h, w):
    r = np.random.default_rng(h * w)
    rng = r.integers(0, 40000, (h, w), dtype=np.uint32)
    sig = r.integers(0, 1 << 16, (h, w), dtype=np.uint16)
    f32 = r.uniform(-1e4, 1e4, (h, w)).astype(np.float32)
    f32.reshape(-1)[::11] = np.nan
    m = (r.random((h, w)) < 0.5).astype(np.uint8)
    shifts = r.integers(-30, 31, h).astype(np.int32)
    inp = tmp_path / "in.bin"
    inp.write_bytes(rng.tobytes() + sig.tobytes() + f32.tobytes() + m.tobytes() + shifts.tobytes())
    out_bin = tmp_path / "out.bin"
    run = subprocess.run([build_example(tmp_path), str(h), str(w), str(inp), str(out_bin)], capture_output=True,
                         text=True, timeout=300)
    assert run.returncode == 0, run.stderr + run.stdout
    lines = run.stdout.splitlines()
    assert lines == ["Only PIXEL_FIELD frame fields are supported here; requested non-pixel fields: [COL]",
                     "Field 'NOPE' not found in LidarFrame.",
                     "coord_2d == x must be either 'u' or 'v'",
                     "invalid value cannot be represented in the field's type",
                     "beam indices can't contain duplicates",
                     "factor == 3 must be a divisor of 8",
                     "FRAME OPS DROPIN OK"]
    o = ofo.Frame(h, w, shifts)
    o.add("RANGE", rng.copy())
    o.add("SIGNAL", sig.copy())
    o.add("F32", f32.copy())
    o.add("COL", np.arange(w, dtype=np.uint32) * 3 + 1, field_class=ofo.COLUMN_FIELD)
    ofo.clip(o, ["RANGE"], 100, 30000, 7)
    ofo.filter_field(o, "SIGNAL", 1000, 20000, 1.7)
    ofo.filter_uv(o, "v", w // 4, w // 2, 9)
    ofo.mask(o, [], m)
    got = out_bin.read_bytes()
    n = h * w
    g_rng = np.frombuffer(got, np.uint32, n, 0).reshape(h, w)
    g_sig = np.frombuffer(got, np.uint16, n, 4 * n).reshape(h, w)
    g_f32 = np.frombuffer(got, np.float32, n, 6 * n).reshape(h, w)
    g_sel = np.frombuffer(got, np.uint32, 3 * w, 10 * n).reshape(3, w)
    assert np.array_equal(g_rng, o.field("RANGE"))
    assert np.array_equal(g_sig, o.field("SIGNAL"))
    assert np.array_equal(g_f32.view(np.uint32), o.field("F32").view(np.uint32))
    assert np.array_equal(g_sel, o.field("RANGE")[[h - 1, 0, h // 2]])
