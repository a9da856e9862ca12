"""H100 drop-in for the ``pointnet2_ops`` package: only ``pointnet2_ops.pointnet2_utils`` and the four functions the
BUFFER-X reference calls (see that module).  Needs the repository root on ``sys.path`` as well (it imports
``bufferx_b200.ops``)."""
