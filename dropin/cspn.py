"""Drop-in for the reference's `models/cspn.py`: put this directory on sys.path BEFORE the reference's ./models
(train.py:64 / eval.py:52 append it, so any earlier entry wins) and `import cspn as post_process`
(torch_resnet_cspn_nyu.py:12) resolves to the H100 implementation.  See INTEGRATION.md."""
from cspn_b200.cspn import Affinity_Propagate  # noqa: F401
