"""cspn_b200: H100-native CSPN propagation (2D 3x3 / 3D 3x3x3) behind the reference's module surface."""
from ._lib import ALGO_AUTO, ALGO_CLUSTER, ALGO_GENERIC, CspnError, describe_plan  # noqa: F401
from .cspn import (Affinity_Propagate, Affinity_Propagate3D, propagate2d, propagate3d)  # noqa: F401
from . import metrics  # noqa: F401

__version__ = '0.1.0'
