"""cspn_b200: H100-native CSPN propagation (2D 3x3, 5x5, 7x7 and CSPN++'s weighted sum of the steps, NLSPN's non-local
propagation with learned per-pixel offsets, PENet's dilated CSPN++ with a learned confidence, DySPN's dynamic propagation
with per-step ring attention, SPN's linear three-way scans, Paddle own-location gates in 2D / 3D 3x3x3, 5x5x5, and the Paddle op with caller-supplied
gates), the guidance / depth heads that feed it
(Unpool + crop + 3x3 convolution in one kernel), the Paddle module's resize_trilinear, the CSPN stereo network's affinity
spatial pyramid pooling, atrous spatial pyramid pooling and fusion, the stereo cost volumes (concatenation and group-wise
correlation) and the disparity regression that consumes them, behind the reference's module surface."""
from ._lib import ALGO_AUTO, ALGO_CLUSTER, ALGO_GENERIC, CspnError, describe_plan  # noqa: F401
from .cspn import (Affinity_Propagate, Affinity_Propagate2DPaddle, Affinity_Propagate3D, Affinity_Propagate3DK,  # noqa: F401
                   Affinity_PropagateDilated, Affinity_PropagateDynamic, Affinity_PropagateK, Affinity_PropagateLinear, Affinity_PropagateNonLocal, Simple_Gudi_UpConv_Block_Last_Layer, affinity_atrous_pool2d, affinity_fuse2d,
                   affinity_pool2d, affinity_propagate, build_concat_volume, build_gwc_volume, disparity_regression, propagate2d,
                   propagate2d_aggregate, propagate2d_dilated, propagate2d_dynamic, propagate2d_k, propagate2d_linear, propagate2d_nonlocal, propagate2d_paddle, propagate3d, propagate3d_k, resize_trilinear, unpool_conv3x3)
from . import metrics  # noqa: F401

__version__ = '0.1.0'
