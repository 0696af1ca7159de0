import sys, torch
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
from dmnerf_b200 import synth
from dmnerf_b200.autograd import mlp_forward_points
from dmnerf_b200.testing import make_models
dev = "cuda"
_, nf, _, _ = make_models(101, 202, 13, dev)
n = 132 * 128 * 96          # 96 tiles per CTA
pts = (torch.rand(n, 3, device=dev) * 6 - 3)
with torch.no_grad():
    for _ in range(3): out = mlp_forward_points(nf, pts)
    torch.cuda.synchronize()
    for reps in (5, 150, 600):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps): out = mlp_forward_points(nf, pts)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        print("reps %d: %.3f ms per launch, %.1f algorithmic TFLOP/s" % (reps, ms, 2.0 * synth.macs_per_sample(13) * n / (ms * 1e-3) / 1e12))
