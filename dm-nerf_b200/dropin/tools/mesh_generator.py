"""Drop-in for tools/mesh_generator.py: `mesh_main` (same signature) on the native kernels; skimage, trimesh (only for the scene's
oriented bounds) and open3d are not needed."""
from dmnerf_b200.mesh import mesh_main  # noqa: F401
