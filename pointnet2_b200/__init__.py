"""pointnet2_b200 — Hopper (sm_90a) PointNet++ set-abstraction / feature-propagation
geometry ops behind the reference's own Python op signatures.

Drop-in for charlesq34/pointnet2's tf_ops/{sampling,grouping,3d_interpolation}:

    from pointnet2_b200.tf_sampling import farthest_point_sample, gather_point
    from pointnet2_b200.tf_grouping import query_ball_point, group_point, knn_point
    from pointnet2_b200.tf_interpolate import three_nn, three_interpolate
    from pointnet2_b200.pointnet_util import sample_and_group, sample_and_group_all, ...

Host code is Python (torch tensors as device buffers) calling hand-written CUDA kernels through a
C-ABI shared library (include/pn2_api.h) with ctypes.  There is no CPU fallback.
"""
from . import _lib  # noqa: F401  (does not load the library until an op is called)
from .tf_sampling import farthest_point_sample, farthest_point_sample_and_gather, gather_point, prob_sample  # noqa: F401
from .tf_grouping import group_point, knn_point, query_ball_point, select_top_k  # noqa: F401
from .tf_interpolate import fp_interpolate_concat, three_interpolate, three_nn, three_nn_interpolate  # noqa: F401
from .sa_layer import SetAbstractionDevice, ball_group, sample_group, sample_group_msg  # noqa: F401
from .pointnet_util import (  # noqa: F401
    group_and_concat,
    pointnet_fp_module,
    pointnet_sa_module,
    pointnet_sa_module_msg,
    sample_and_group,
    sample_and_group_all,
)
from .host import SetAbstractionHost, SetAbstractionPipeline  # noqa: F401
from .layers import batch_invariant, is_batch_invariant  # noqa: F401
from .render import project_points, render_balls, show_points  # noqa: F401
from . import _ops  # noqa: F401  (registers the pn2:: torch operators; loads nothing)

__version__ = "0.1.0"
