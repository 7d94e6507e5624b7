"""Every kernel of the library is launched through ob::launch, which counts it in its family: no `<<<` outside
that helper's definition in ob_internal.h, and no hand-kept launch tallies.  Per-call device memory comes from one
typed Staging, and every CUB device-wide call goes through the helper in ob_cub.cuh that takes its temporary storage
from there."""
import os
import re

import __graft_entry__ as graft

CSRC = os.path.join(graft.ROOT, "ouster-sdk_b200", "csrc")


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, f.read()


def test_every_kernel_launch_goes_through_the_launch_helper():
    found = {name: src.count("<<<") for name, src in _sources() if "<<<" in src}
    assert found == {"ob_internal.h": 1}, found
    helper = dict(_sources())["ob_internal.h"]
    assert re.search(r"void launch\(int family, void \(\*kernel\)\(P\.\.\.\), dim3 grid, dim3 block, size_t smem, "
                     r"cudaStream_t st, A&&\.\.\. args\) \{\n\s*kernel<<<grid, block, smem, st>>>", helper)


def test_no_hand_kept_launch_counts():
    assert [name for name, src in _sources() if "count_launch" in src] == []


def test_cub_device_calls_go_through_the_cub_helper():
    assert [name for name, src in _sources() if "cub::Device" in src] == ["ob_cub.cuh"]


def test_one_typed_staging():
    srcs = dict(_sources())
    assert [name for name, src in srcs.items() if "scratch(stg," in src] == []
    assert [name for name, src in srcs.items() if re.search(r"auto alloc = \[", src)] == []
    common = srcs["ob_api_common.h"]
    staging = common[common.index("class Staging {"):common.index("};", common.index("class Staging {"))]
    assert "void**" not in staging
    assert [name for name, src in srcs.items() if re.search(r"if \(e == cudaSuccess[^)]*\) e = (stg|res)\.", src)] == []
