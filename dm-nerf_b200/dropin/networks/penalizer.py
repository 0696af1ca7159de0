"""networks.penalizer (reference networks/penalizer.py) on the native kernels: same two names, same signatures."""
from dmnerf_b200.penalizer import emptiness_penalizer, ins_penalizer   # noqa: F401
