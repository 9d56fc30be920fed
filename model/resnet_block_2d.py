"""Drop-in for /root/reference/model/resnet_block_2d.py (channels-last H100 implementation)."""
from ctrl_adapter_b200.layers import ResnetBlock2D  # noqa: F401
