"""ConditionalWaveFlow.infer at cfg4 shapes: CUDA-event time of a graph replay (third call of the same shape)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parakeet_b200.models import ConditionalWaveFlow
dev = "cuda"
B, FRAMES = 16, 400
CH = int(os.environ.get("PK_WF_CHANNELS", "64"))      # 128 = examples/waveflow/config.py
wf = ConditionalWaveFlow([16, 16], 8, 8, 16, CH, 80, (3, 3), device=dev, seed=4)
g = torch.Generator().manual_seed(4)
mel = (torch.randn(B, 80, FRAMES, generator=g) * 0.5 - 3).to(dev)
z = torch.randn(B, 256 * FRAMES - 272, generator=g).to(dev)
for _ in range(3):
    y = wf.infer(mel, z=z)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(3):
    y = wf.infer(mel, z=z)
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 3
print(f"waveflow {CH} ch b16 x 400 frames: {ms:.1f} ms/call, "
      f"{y.numel() / ms * 1e3 / 1e6:.2f} M samples/s, replays {wf._graphs.replays}, finite {bool(torch.isfinite(y).all())}", flush=True)
