"""GPU diagnostic for pk_conv_gemm: wgmma path vs SIMT path vs torch fp64 (prints error tables)."""
import sys, os, math
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from parakeet_b200 import ops

torch.manual_seed(0)
dev = "cuda"

def ref_conv(x, w, bias, taps, dil, pad, act, residual, lens, scale=1.0):
    # x (B,T,C) f64, w [n, C, taps]
    y = F.conv1d(x.transpose(1, 2), w, None, padding=0 if taps == 1 else pad * dil, dilation=dil).transpose(1, 2) * scale
    if bias is not None: y = y + bias
    if act == "relu": y = torch.relu(y)
    if act == "tanh": y = torch.tanh(y)
    if residual is not None: y = y + residual
    if lens is not None:
        m = torch.arange(y.shape[1], device=y.device)[None, :, None] < lens[:, None, None]
        y = y * m
    return y

def err(a, b):
    return ((a.double() - b.double()).abs().max() / b.abs().max().clamp_min(1e-30)).item()

def run(name, B, T, Cin, N, taps=1, dil=1, bias=True, act=None, res=False, lens=False, passes=3):
    x = torch.randn(B, T, Cin, device=dev)
    w = torch.randn(N, Cin, taps, device=dev) / math.sqrt(Cin * taps)
    b = torch.randn(N, device=dev) if bias else None
    r = torch.randn(B, T, N, device=dev) if res else None
    ln = torch.randint(T // 2, T + 1, (B,), device=dev, dtype=torch.int32) if lens else None
    xs = ops.Split.from_f32(x)
    ws = ops.pack_weight(w, dev)
    pad = (taps - 1) // 2
    yref = ref_conv(x.double(), w.double(), b.double() if bias else None, taps, dil, pad, act,
                    r.double() if res else None, ln, 1.0)
    out = {}
    for mode, simt in (("tc", False), ("simt", True)):
        y, ys = ops.conv_gemm(xs, ws, n=N, k=Cin, taps=taps, dil=dil, bias=b, act=act, residual=r, lens=ln,
                              out_f32=True, out_split=True, passes=passes, simt=simt)
        torch.cuda.synchronize()
        out[mode] = (err(y, yref), err(ys.float(), yref))
    print(f"{name:34s} B{B} T{T} C{Cin} N{N} taps{taps} dil{dil} p{passes}: tc f32 {out['tc'][0]:.2e} split {out['tc'][1]:.2e} | "
          f"simt f32 {out['simt'][0]:.2e}", flush=True)
    return out['tc'][0]

print("split roundtrip:", err(ops.Split.from_f32(torch.randn(1000, 37, device=dev)).float(),
                              torch.randn(1, device=dev) * 0 + ops.Split.from_f32(torch.randn(1000, 37, device=dev)).float()))
x = torch.randn(5, 1000, 37, device=dev)
print("split error vs f32:", err(ops.Split.from_f32(x).float(), x))
bad = 0
cases = [
    ("linear 64->64 one tile", 1, 128, 64, 64),
    ("linear 64->128", 1, 128, 64, 128),
    ("linear 128->128 2 chunks", 1, 128, 128, 128),
    ("linear 384->384", 2, 300, 384, 384),
    ("linear 384->1152", 2, 300, 384, 1152),
    ("linear 384->80 partial N", 2, 300, 384, 80),
    ("linear 80->256 partial K", 2, 300, 80, 256),
]
for c in cases:
    e = run(*c); bad += e > 1e-4
e = run("conv k3 384->1536 relu", 2, 300, 384, 1536, taps=3, act="relu"); bad += e > 1e-4
e = run("conv k3 1536->384 +res +lens", 2, 300, 1536, 384, taps=3, res=True, lens=True); bad += e > 1e-4
e = run("conv k5 80->256 tanh", 2, 333, 80, 256, taps=5, act="tanh", bias=True); bad += e > 1e-4
e = run("dilated k3 d8 64->128", 2, 1000, 64, 128, taps=3, dil=8); bad += e > 1e-4
e = run("dilated k3 d512 64->128", 1, 3000, 64, 128, taps=3, dil=512); bad += e > 1e-4
e = run("linear 384->384 1 pass", 2, 300, 384, 384, passes=1); 
print("single-pass bf16 error (expected ~1e-2..1e-3):", e)

# attention-like batched NT matmul: S[b,h] = Q[b,h] K[b,h]^T / sqrt(dk)
B, T, H, dk = 2, 200, 2, 192
qkv = torch.randn(B, T, 3 * H * dk, device=dev)
qs = ops.Split.from_f32(qkv)
Tp = (T + 63) // 64 * 64
S = torch.zeros(B, H, T, Tp, device=dev)
spec_q = dict(rows=T, cols=3 * H * dk, ld=3 * H * dk, batch_stride=T * 3 * H * dk, batches=B, bmul=1, hmul=0, col0=0, colh=dk)
spec_k = dict(rows=T, cols=3 * H * dk, ld=3 * H * dk, batch_stride=T * 3 * H * dk, batches=B, bmul=1, hmul=0, col0=H * dk, colh=dk)
ops.batched_matmul_nt(qs, qs, batch=B, heads=H, m=T, n=T, k=dk, a_spec=spec_q, b_spec=spec_k, scale=1 / math.sqrt(dk),
                      y_f32=S, y_batch_stride=H * T * Tp, y_head_stride=T * Tp, y_ld=Tp)
torch.cuda.synchronize()
q = qkv[..., :H * dk].reshape(B, T, H, dk).permute(0, 2, 1, 3).double()
k = qkv[..., H * dk:2 * H * dk].reshape(B, T, H, dk).permute(0, 2, 1, 3).double()
Sref = q @ k.transpose(-1, -2) / math.sqrt(dk)
e = err(S[..., :T], Sref); print("attention scores QK^T:", e); bad += e > 1e-4
print("pad cols zero:", S[..., T:].abs().max().item())
print("launches", ops._lib.launch_count())
print("FAILED" if bad else "ALL OK", bad)
sys.exit(1 if bad else 0)
