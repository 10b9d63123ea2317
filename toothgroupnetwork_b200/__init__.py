"""toothgroupnetwork_b200 -- H100-native (sm_90a) point-cloud sampling / neighbour-search /
grouping / interpolation / grouped shared-MLP operators behind the operator API of
limhoyeon/ToothGroupNetwork's ``external_libs/pointops`` and ``external_libs/pointnet2_utils``.

Importing the package does not touch the GPU; the CUDA library is loaded on first use and
its absence is a hard error (there is no CPU or PyTorch fallback)."""
__version__ = "0.1.0"
