"""Every kernel of the library is launched through ob::launch, which counts it in its family: no `<<<` outside
that helper's definition in ob_internal.h, and no hand-kept launch tallies."""
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
