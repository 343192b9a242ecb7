"""event_utils_b200 -- H100-native (sm_90a) drop-in for the data-parallel hot path of
TimoStoff/event_utils: event -> voxel grid / event image binning and the contrast-maximisation
inner loop.  Same Python function signatures as the reference; the work is done by hand-written
CUDA kernels in libevk.so (C ABI: include/evk.h).  No CPU fallback.

Module map (reference module -> this package):
    lib/representations/voxel_grid.py -> event_utils_b200.representations.voxel_grid
    lib/representations/image.py      -> event_utils_b200.representations.image
    lib/transforms/optic_flow.py      -> event_utils_b200.transforms.optic_flow
    lib/contrast_max/warps.py         -> event_utils_b200.contrast_max.warps
    lib/contrast_max/objectives.py    -> event_utils_b200.contrast_max.objectives
    lib/contrast_max/events_cmax.py   -> event_utils_b200.contrast_max.events_cmax (drivers)
    lib/util/event_util.py (mask)     -> event_utils_b200.util.event_util
    lib/data_loaders (window tables, RobustNorm) -> event_utils_b200.data_loaders.{windows,data_augmentation}
    multi-GPU (no reference counterpart)         -> event_utils_b200.parallel
"""
from . import config  # noqa: F401

__version__ = "0.1.0"
