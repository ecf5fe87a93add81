"""camlasercalibratool_b200 -- H100-native (sm_90a) camera<-laser extrinsic solve.

The product is libclc_b200.so (C ABI in include/clc_b200.h, CUDA in csrc/).  This package holds the build recipe,
the ctypes binding and a Python mirror of the reference's solver interface (api.py).  Nothing here falls back to
the CPU: importing is cheap, but every numeric call needs the CUDA library and an H100.
"""
from . import _build  # noqa: F401
from .api import (  # noqa: F401
    CamLaserCalClosedSolution,
    CamLaserCalibration,
    LineFittingCeres,
    ClcError,
    Comm,
    FRAME_ROW_DTYPE,
    Group,
    Oberserve,
    Problem,
    QUANTILES_MAX,
    Selection,
    T_to_pose7,
    comm_unique_id,
    debug_pack,
    default_options,
    frame_influence,
    launch_count,
    marshal,
    pose7_to_T,
    select_frames_from_report,
    shard_range,
    upload_stats,
)

__all__ = [
    "CamLaserCalClosedSolution", "CamLaserCalibration", "LineFittingCeres", "ClcError", "Comm", "Group", "Oberserve", "Problem", "T_to_pose7",
    "comm_unique_id", "default_options", "launch_count", "marshal", "pose7_to_T", "shard_range", "debug_pack", "upload_stats",
    "FRAME_ROW_DTYPE", "frame_influence", "Selection", "select_frames_from_report",
    "QUANTILES_MAX",
]
