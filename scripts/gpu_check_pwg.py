"""GPU diagnostic: PWG generator (CUDA) vs the torch-CPU oracle at small sizes, plus a timing of cfg2."""
import sys, os, math, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from oracle import pwg as opwg
from parakeet_b200.models import PWGGenerator

dev = "cuda"
def err(a, b):
    return ((a.double().cpu() - b.double().cpu()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()

cfg = dict(opwg.DEFAULT_GENERATOR_PARAMS)
params = opwg.synth_params(2, weight_norm=True)
gen = PWGGenerator(**cfg, device=dev)
gen.set_state_dict(params)
folded = opwg.fold_weight_norm(params)

# 1. upsample net alone
x, c = opwg.synth_inputs(2, batch=2, mel_frames=40)
with torch.no_grad():
    c_ref = opwg.conv_in_upsample_net(folded, c, cfg["upsample_scales"])
c_gpu = gen.upsample(c.to(dev))
torch.cuda.synchronize()
print("upsample net err:", err(c_gpu, c_ref), flush=True)

# 2. full generator, small
with torch.no_grad():
    y_ref, inter = opwg.generator_forward(folded, x, c, return_intermediates=True)
y = gen(x.to(dev), c.to(dev))
torch.cuda.synchronize()
print("x30 err:", err(gen._last_x.float().transpose(1, 2), inter["x_layers"][-1]))
print("skip err (incl. deferred bias):", err((gen._ws[(2, 12000)]["skip"] + gen._pack()["skip_bias_sum"]).transpose(1, 2) * math.sqrt(1 / 30), inter["skips"]))
e = err(y, y_ref)
print("generator out err:", e, "shape", tuple(y.shape), flush=True)
bad = e > 1e-3

# 3. remove_weight_norm path gives the same
gen.remove_weight_norm()
y2 = gen(x.to(dev), c.to(dev)); torch.cuda.synchronize()
print("after remove_weight_norm, max diff:", (y2 - y).abs().max().item())

# 4. ragged batch with lens == per-utterance runs
frames = [40, 25, 33]
hop = 300
Tmax = max(frames) * hop
xs = torch.zeros(3, 1, Tmax); cs = torch.zeros(3, 80, max(frames) + 4)
refs = []
for i, f in enumerate(frames):
    xi, ci = opwg.synth_inputs(10 + i, batch=1, mel_frames=f)
    xs[i, :, :f * hop] = xi[0]; cs[i, :, :f + 4] = ci[0]
    # the batched conditioning beyond the utterance end must look like the single-utterance replicate padding
    cs[i, :, f + 4:] = 0
    with torch.no_grad():
        refs.append(opwg.generator_forward(folded, xi, ci)[0])
lens = torch.tensor([f * hop for f in frames], dtype=torch.int32, device=dev)
yb = gen(xs.to(dev), cs.to(dev), lens=lens); torch.cuda.synchronize()
for i, f in enumerate(frames):
    e = err(yb[i, :, :f * hop], refs[i]); bad |= e > 1e-3
    print(f"ragged utt {i} ({f} frames) err: {e:.3e}")

# 5. inference() API vs oracle
mel = torch.randn(30, 80); noise = torch.randn(1, 1, 30 * hop)
with torch.no_grad():
    r = opwg.generator_inference(folded, mel, noise)
o = gen.inference(mel.to(dev), x=noise.to(dev)); torch.cuda.synchronize()
e = err(o, r); bad |= e > 1e-3
print("inference() err:", e, tuple(o.shape))

# 6. timing at cfg2 (B=32, 400 frames)
if "--time" in sys.argv:
    x, c = opwg.synth_inputs(2, batch=32, mel_frames=400)
    x, c = x.to(dev), c.to(dev)
    for _ in range(2): y = gen(x, c)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    n = 3
    ev[0].record()
    for _ in range(n): y = gen(x, c)
    ev[1].record(); torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / n
    print(f"cfg2: {ms:.2f} ms per batch -> {32 * 120000 / ms / 1e3:.1f} M samples/s", flush=True)
    # check a slice against the oracle run on utterance 0 only (CPU ~1-2 s per utterance-second)
    with torch.no_grad():
        r0 = opwg.generator_forward(folded, x[:1, :, :].cpu(), c[:1].cpu())
    e = err(y[:1], r0); bad |= e > 1e-3; print("cfg2 utt0 err:", e)
print("FAILED" if bad else "ALL OK")
sys.exit(1 if bad else 0)
