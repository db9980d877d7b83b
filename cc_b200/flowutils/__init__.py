"""The reference's flowutils import paths: flowlib (Middlebury colours on the device) and flow_io (KITTI / .flo files)."""
from . import flow_io, flowlib      # noqa: F401
