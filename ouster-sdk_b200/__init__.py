"""ouster-sdk_b200: CUDA (H100) scan -> pointcloud path (decode -> destagger -> cartesian).

Python host mirror over the C ABI (include/ouster_b200.h).  The directory name carries a
hyphen (it is the name the build contract fixes), so import it through
`__graft_entry__.load_package()` which registers it as module `ouster_sdk_b200`.
"""
from . import _capi  # noqa: F401  (fails loudly when the CUDA library is not built)
from .core import (Decoder, Stream, XYZLut, XYZLutFloat, XYZLutT, cartesian, destagger, dewarp, dewarp_frame, dewarp_frames, normals, transform, voxel_downsample, VoxelMap, icp_align, map_rows, icp_linear_system, cloud_align, cloud_nearest, zone_render, ZoneMonitor, ImageProcessor, scan_to_cloud, plan_scan_to_cloud,  # noqa: F401
                   device_count, kernel_launch_count, pinned_empty, set_tunable)
from .host import get_device, set_device  # noqa: F401,E402
from .host import FrameBatcher, FramePipeline, PcapLidarSource, LidarFrame, LidarScan, ScanBatcher, SensorInfo, frame_to_packets  # noqa: F401,E402
from . import sharding  # noqa: F401,E402
from . import pyapi  # noqa: F401,E402
from . import frame_ops  # noqa: F401,E402
