"""Drop-in for the reference's `models` package (reference models/__init__.py:1-2):
`models.DispResNet(num_layers, pretrained)` and `models.PoseResNet(num_layers, pretrained)` with the
reference's state_dict keys, executed by hand-written sm_90a kernels (scsfm/nets.py)."""
from scsfm.nets import DispResNet, PoseResNet, ResnetEncoder  # noqa: F401
