"""Time TransformerTTS.inference at the ljspeech recipe config on one GPU: B = 1, a 150-token text + eos, prob threshold 2 so that
maxlen stops the loop after a fixed number of steps.  The per-step cost is the slope between a 100-step and an 800-step run (the
encoder, the K / V GEMM and the postnet cancel); weight bytes per step count every fp32 decoder weight the step reads once.
Also: the teacher-forced forward at the recipe batch (16 ragged utterances, up to 800 frames), and for context the eager fp32 torch
decoder step of the reference (forward_one_step: the prenet over every earlier frame, then each layer's new row over its cached
outputs) on the same card with TF32 off, at step 400.
Prints one JSON line, with the card's name, power limit and max SM clock read in the same run.

    python scripts/time_transformer_tts.py
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle.fastspeech2 as ofs  # noqa: E402
import oracle.transformer_tts as ot  # noqa: E402
from parakeet_b200.models import TransformerTTS  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps * 1e3          # us per call


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    cfg, seed = ot.GOLDEN_CONFIGS["ljspeech"]
    kw = {k: v for k, v in cfg.items() if k not in ("idim", "odim")}
    dev = torch.device("cuda:0")
    m = TransformerTTS(cfg["idim"], cfg["odim"], device=dev, **kw)
    m.set_state_dict(ot.synth_params(seed, cfg))
    text = ot.golden_text(cfg, 1, 150).to(dev)
    T = 151
    run = lambda n: (lambda: m.inference(text, threshold=2.0, maxlenratio=(n + 0.5) / T, seed=1))  # noqa: E731
    t100, t800 = timed(run(100), 5), timed(run(800), 3)
    step_us = (t800 - t100) / 700
    A, U, Up, L, odim = cfg["adim"], cfg["dunits"], cfg["dprenet_units"], cfg["dlayers"], cfg["odim"]
    weights = L * (6 * A * A + 2 * A * U) + Up * odim + Up * Up + A * Up + A * (odim + 1)
    # the teacher-forced forward: 16 utterances, text 60..150 tokens, 500..800 frames
    g = torch.Generator().manual_seed(3)
    tl = torch.randint(60, 151, (16,), generator=g)
    sl = torch.randint(500, 801, (16,), generator=g)
    tb = torch.randint(1, cfg["idim"] - 1, (16, int(tl.max())), generator=g).to(dev)
    sp = (torch.randn(16, int(sl.max()), cfg["odim"], generator=g) * 0.5).to(dev)
    fwd_ms = timed(lambda: m(tb, tl.to(dev), sp, sl.to(dev), seed=1), 5) / 1e3
    # the eager fp32 step at position 400
    torch.backends.cuda.matmul.allow_tf32 = False
    p = {k: v.to(dev) for k, v in ot.synth_params(seed, cfg).items()}
    t = 400
    with torch.no_grad():
        p_cpu = ot.synth_params(seed, cfg)
        hs = ot.encode(p_cpu, cfg, torch.cat([text.cpu(), torch.tensor([cfg["idim"] - 1])]).unsqueeze(0)).to(dev)
        pe = ofs.positional_encoding(t + 1, A).to(dev)
        ys = torch.randn(1, t + 1, odim, device=dev)
        cache = [torch.randn(1, t, A, device=dev) for _ in range(L)]
        keep = (torch.rand(cfg["dprenet_layers"], 1, t + 1, Up, device=dev) >= 0.5).float()

        def eager_step():
            h = ys
            for i in range(cfg["dprenet_layers"]):
                h = torch.relu(ofs.linear(p, f"decoder.embed.0.0.prenet.{i}.0", h)) * keep[i] * 2.0
            x = ofs.linear(p, "decoder.embed.0.1", h) + p["decoder.embed.1.alpha"] * pe
            for l in range(L):
                q = f"decoder.decoders.{l}."
                tn = ofs.layer_norm(p, q + "norm1", x)
                y = x[:, -1:] + ot._mha(p, q + "self_attn.", tn[:, -1:], tn, cfg["aheads"])[0]
                y = y + ot._mha(p, q + "src_attn.", ofs.layer_norm(p, q + "norm2", y), hs, cfg["aheads"])[0]
                y = y + ofs.linear(p, q + "feed_forward.w_2", torch.relu(ofs.linear(p, q + "feed_forward.w_1", ofs.layer_norm(p, q + "norm3", y))))
                x = torch.cat([cache[l], y], 1)
            z = ofs.layer_norm(p, "decoder.after_norm", x[:, -1])
            return ofs.linear(p, "feat_out", z), torch.sigmoid(ofs.linear(p, "prob_out", z))

        eager_us = timed(eager_step, 20)
    print(json.dumps({"card": card(), "config": "ljspeech", "T_enc": T, "inference_100_steps_ms": round(t100 / 1e3, 2),
                      "inference_800_steps_ms": round(t800 / 1e3, 2), "us_per_decoder_step": round(step_us, 1),
                      "weight_MB_per_step": round(4 * weights / 1e6, 1), "weight_GB_per_s": round(4 * weights / step_us / 1e3, 1),
                      "forward_b16_ms": round(fwd_ms, 1), "forward_frames": int(sl.sum()), "eager_fp32_step_at_400_us": round(eager_us, 1)}))


if __name__ == "__main__":
    main()
