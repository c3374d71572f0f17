"""`from ops.voxel_pooling import voxel_pooling` (lss.py:14) — same call, H100-native kernel underneath."""
from .voxel_pooling import voxel_pooling, VoxelPooling, last_pos_memo  # noqa: F401
