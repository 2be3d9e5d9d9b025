"""cspn_b200: H100-native CSPN propagation (2D 3x3, 5x5, 7x7, Paddle own-location gates
in 2D / 3D 3x3x3, 5x5x5, and the Paddle op with caller-supplied gates) and the guidance / depth heads that feed it
(Unpool + crop + 3x3 convolution in one kernel) behind the reference's module surface."""
from ._lib import ALGO_AUTO, ALGO_CLUSTER, ALGO_GENERIC, CspnError, describe_plan  # noqa: F401
from .cspn import (Affinity_Propagate, Affinity_Propagate2DPaddle, Affinity_Propagate3D, Affinity_Propagate3DK,  # noqa: F401
                   Affinity_PropagateK, Simple_Gudi_UpConv_Block_Last_Layer, affinity_propagate, propagate2d, propagate2d_k,
                   propagate2d_paddle, propagate3d, propagate3d_k, unpool_conv3x3)
from . import metrics  # noqa: F401

__version__ = '0.1.0'
