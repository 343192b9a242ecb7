"""Contrast maximisation: motion models (`warps`), objectives evaluated by the fused GPU pass
(`objectives`), the optimiser / grid-search drivers around them (`events_cmax`) and the batched,
differentiable losses of the dense flow (`flow_objective`, and the average-timestamp loss of
`flow_timestamp_objective`) and of the parametric models (`motion_objective`, and the average-timestamp
loss of `motion_timestamp_objective`), the batched fits of one motion per window to the contrast loss
(`motion_fit`) and to the average-timestamp loss (`motion_timestamp_fit`), and the segmentation of every
window into several motions (`motion_segmentation`), and the loss, candidates pass and coarse-to-fine fit of a dense
flow given on a grid of nodes, to the contrast loss (`grid_flow`) and to the average-timestamp loss
(`grid_flow_timestamp`), and of an inverse-depth field on a grid of nodes under a known camera motion, to the
contrast loss (`depth_grid`) and to the average-timestamp loss (`depth_grid_timestamp`), and of the camera motion and
such a field together (`motion_and_depth`).  The batched losses share their
event preparation, argument checks and loops over chunks of windows (`_batched`).

Everything public in the fifteen modules is re-exported here, so `from event_utils_b200.contrast_max
import linvel_warp, variance_objective, optimize_contrast` works the way the same import from the
reference's `lib.contrast_max` package does.
"""
from . import depth_grid as _depth_grid
from . import depth_grid_timestamp as _depth_grid_timestamp
from . import events_cmax as _drivers
from . import flow_objective as _flow_objective
from . import flow_timestamp_objective as _flow_timestamp_objective
from . import grid_flow as _grid_flow
from . import grid_flow_timestamp as _grid_flow_timestamp
from . import motion_and_depth as _motion_and_depth
from . import motion_fit as _motion_fit
from . import motion_objective as _motion_objective
from . import motion_segmentation as _motion_segmentation
from . import motion_timestamp_fit as _motion_timestamp_fit
from . import motion_timestamp_objective as _motion_timestamp_objective
from . import objectives as _objectives
from . import warps as _warps

for _module in (_drivers, _warps, _objectives, _flow_objective, _flow_timestamp_objective, _motion_objective,
                _motion_timestamp_objective, _motion_fit, _motion_timestamp_fit, _motion_segmentation, _grid_flow,
                _grid_flow_timestamp, _depth_grid, _depth_grid_timestamp, _motion_and_depth):
    globals().update({_name: getattr(_module, _name) for _name in dir(_module) if not _name.startswith("_")})
del _module
