"""dm-nerf_b200: H100-native fused volumetric renderer behind DM-NeRF's Python call surface.

Import as `dmnerf_b200` (see ../dmnerf_b200/__init__.py).  Nothing here imports oracle/.
Heavy submodules (anything touching the CUDA library) are imported lazily so that CPU-only
tooling (synth, build) works without a GPU.
"""
__version__ = "0.1.0"
