"""kiss_icp_b200 — CUDA (H100, sm_90a) implementation of KISS-ICP's per-scan registration hot
path behind the reference's own Python surface (python/kiss_icp/*.py). The compute lives in
hand-written CUDA kernels reached through the C-ABI of include/kiss_icp_b200.h; this package
is the host-side mirror of the reference interface. No CPU fallback."""
from .config import KISSConfig, load_config  # noqa: F401
from .constraints import RECOMMENDED_DEGENERACY_RATIO, Constraints, ScanDegeneracy, covariance, degeneracy  # noqa: F401
from .free_space import FreeSpace, FreeSpaceParams  # noqa: F401
from .kiss_icp import KissICP  # noqa: F401
from .mapping import VoxelHashMap, get_voxel_hash_map  # noqa: F401
from .places import PlaceDatabase, PlaceDescriptorParams, PlaceMatch, PlaceRelocalizationResult  # noqa: F401
from .pose_graph import PoseGraph, PoseGraphFactorInfo, PoseGraphOptions, PoseGraphReport  # noqa: F401
from .pose_graph import PlaneAdjustmentParams, PlaneAdjustmentReport, PlaneRound  # noqa: F401
from .loop_closure import LoopCloser, LoopClosure, SessionMatch, SessionMerge, SessionMergeReport, session_consensus  # noqa: F401
from .preprocess import Preprocessor, get_preprocessor  # noqa: F401
from .registration import Registration, get_registration  # noqa: F401
from .relocalization import RelocalizationResult, RelocalizationSearch  # noqa: F401
from .threshold import AdaptiveThreshold, FixedThreshold, get_threshold_estimator  # noqa: F401
from .voxelization import voxel_down_sample  # noqa: F401
from .preprocess import correct_kitti_scan  # noqa: F401
from .metrics import absolute_trajectory_error, sequence_error  # noqa: F401
from .motion import Motion, deskew, motion_from_gyro  # noqa: F401
from .rig import Rig, Sensor, merge_rig  # noqa: F401
from .calibration import RigCalibration, SensorCalibration, calibrate_rig  # noqa: F401
from .calibration import RigClockCalibration, SensorClockCalibration, calibrate_rig_clocks  # noqa: F401

__version__ = "0.1.0"
