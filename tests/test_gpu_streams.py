"""GPU tests of the stream a call on CUDA tensors runs on when no `stream=` is given: the torch current stream of the
tensors' device, through one wrapper per (device, stream) that an earlier call made, so a CUDA graph can capture the
call as it is and the call is ordered after the torch work that wrote its inputs."""
import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import oracle as orc
from tests.test_gpu_align import room_pair, rot
from tests.test_oracle_normals import room_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    graft.build()
    m = graft.load_package()
    assert m.device_count() > 0
    return m


def _replays_bit_identical(call):
    """call() once on a side torch stream, then capture call() on that stream and replay it twice; each replay must
    give the first call's outputs bit for bit."""
    import torch
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        want = call()
        s.synchronize()
        with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
            got = call()
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_icp_align_is_captured_without_a_stream(ob):
    import torch
    dev = torch.device("cuda", 0)
    _, rng, d = room_scene(64, 1024)
    pts = (d * rng[..., None] * 0.001).reshape(-1, 3)
    m = ob.VoxelMap(0.5, 30.0, 20)
    m.add_points(pts)
    step = np.eye(4)
    step[:3, :3] = rot(np.radians([0.0, 0.0, 0.8]))
    step[:3, 3] = [0.04, 0.01, 0.0]
    src = torch.from_numpy(pts[::5] @ step[:3, :3].T + step[:3, 3]).to(dev)
    _replays_bit_identical(lambda: ob.icp_align(m, src, 3.0, 1.0, 50))


def test_cloud_align_is_captured_without_a_stream(ob):
    import torch
    dev = torch.device("cuda", 0)
    src, tgt, ns, nt, _ = room_pair()
    s, t, sn, tn = (torch.from_numpy(a).to(dev) for a in (src, tgt, ns, nt))
    _replays_bit_identical(lambda: ob.cloud_align(s, t, sn, tn))
    _replays_bit_identical(lambda: ob.cloud_align(s, t))


def test_one_wrapper_per_torch_stream(ob):
    import torch
    core = ob.core
    x = torch.zeros(4, device="cuda:0")
    a, b = core._stream_for(x), core._stream_for(x)
    assert a is b and (a.cuda_stream or 0) == torch.cuda.current_stream().cuda_stream   # NULL handle reads as None
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        c = core._stream_for(x)
        assert c is core._stream_for(x) and c is not a and c.cuda_stream == side.cuda_stream
    explicit = ob.Stream(0)
    assert core._stream_for(x, explicit) is explicit
    assert core._stream_for(np.zeros(4)) is core._stream(None, 0)


def test_calls_are_ordered_after_the_torch_work_that_wrote_their_inputs(ob):
    """A range image is written on a side torch stream behind a long GPU wait; cartesian and destagger called on
    that stream must read the written values, with no synchronise between the write and the calls.  Each round
    writes another image; only the first allocates (device memory and the stream's launch tables), which can
    synchronise the device by itself."""
    import torch
    dev = torch.device("cuda", 0)
    h, w = 64, 1024
    rs = np.random.default_rng(11)
    d = (rs.random((h * w, 3)) + 0.5).astype(np.float32)
    o = (rs.random((h * w, 3)) * 0.01).astype(np.float32)
    shifts = rs.integers(-30, 31, size=h).astype(np.int32)
    lut = ob.XYZLutT.from_arrays(d, o, h, w)
    rngs = [rs.integers(0, 1 << 20, size=(h, w), dtype=np.uint32) for _ in range(3)]
    srcs = [torch.from_numpy(a.view(np.int32)).to(dev) for a in rngs]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    for rng, src in zip(rngs, srcs):
        with torch.cuda.stream(side):
            r = torch.zeros((h, w), dtype=torch.int32, device=dev)
            torch.cuda._sleep(50_000_000)          # the copy below lands tens of milliseconds later
            r.copy_(src)
            xyz = ob.cartesian(lut, r.view(torch.uint32))
            img = ob.destagger(r, shifts)
            xyz_h, img_h = xyz.cpu().numpy(), img.cpu().numpy()
        assert np.array_equal(xyz_h, orc.cartesian(rng, d, o))
        assert np.array_equal(img_h.view(np.uint32), orc.destagger(rng, shifts))
        del r, xyz, img                            # the next round reuses these blocks
