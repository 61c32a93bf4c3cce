"""Time TransformerTTSTrainStep.step at the ljspeech recipe (examples/transformer_tts/ljspeech/conf/default.yaml: adim 512,
8 heads, 6 + 6 layers, 1024 units, 5-layer postnet, every dropout rate of the yaml, guided source-attention loss lambda 10, Adam
1e-3) with CUDA events around CUDA-graph replays, after the timed shape has been warmed up (eager, capture, replay).

Workload: the recipe batch of scripts/time_transformer_tts.py - 16 utterances of 60..150 tokens and 500..800 mel frames (about
10 k frames), seeded weights.  Algorithmic TFLOP/s counts 3 x the forward's GEMM FLOP (projections, attention scores and P V,
feed-forward, prenet, output and postnet convolutions) over ALL padded rows, 2 FLOP per multiply-add.

    python scripts/time_transformer_tts_train.py [--steps 10] [--repeats 2] [--profile DIR]

--profile (a separate run: tracing slows the host) writes torch.profiler's kernel table of 3 steps to DIR.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def workload(cfg, dev):
    """16 utterances, text 60..150 tokens, 500..800 frames (the seed and shape of time_transformer_tts.py's forward)."""
    g = torch.Generator().manual_seed(3)
    tl = torch.randint(60, 151, (16,), generator=g)
    sl = torch.randint(500, 801, (16,), generator=g)
    text = torch.zeros(16, int(tl.max()), dtype=torch.int64)
    for b, n in enumerate(tl.tolist()):
        text[b, :n] = torch.randint(1, cfg["idim"] - 1, (n,), generator=g)
    sp = torch.randn(16, int(sl.max()), cfg["odim"], generator=g) * 0.5
    return dict(text=text.to(dev), text_lengths=tl.to(dev), speech=sp.to(dev), speech_lengths=sl.to(dev))


def algorithmic_flop(cfg, B, T, L):
    """Forward GEMM FLOP of one step at text width T (eos included) and L frames, every padded row counted."""
    A, H, U, D, Up, odim = cfg["adim"], cfg["aheads"], cfg["eunits"], cfg["dunits"], cfg["dprenet_units"], cfg["odim"]
    k, dk = cfg["positionwise_conv_kernel_size"], A // H
    enc = cfg["elayers"] * (2 * T * A * 3 * A + 2 * 2 * H * T * T * dk + 2 * T * A * A + 2 * 2 * T * A * U * k)
    mem = 2 * T * A * 2 * A * cfg["dlayers"]
    pre = 2 * L * (odim * Up + (cfg["dprenet_layers"] - 1) * Up * Up + Up * A)
    dec = cfg["dlayers"] * (2 * L * A * 3 * A + 2 * 2 * H * L * L * dk + 2 * L * A * A + 2 * L * A * A + 2 * 2 * H * L * T * dk
                            + 2 * L * A * A + 2 * 2 * L * A * D)
    out = 2 * L * A * (odim + 1)
    n, C, kp = cfg["postnet_layers"], cfg["postnet_chans"], cfg["postnet_filts"]
    post = sum(2 * L * (odim if i == 0 else C) * (odim if i == n - 1 else C) * kp for i in range(n))
    return B * (enc + mem + pre + dec + out + post)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--profile", default=None, help="directory for the torch.profiler table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU and has no CPU fallback")
    from time_transformer_tts import card
    from oracle import transformer_tts as ot
    from parakeet_b200.models import TransformerTTS
    from parakeet_b200.training import TransformerTTSTrainStep
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    cfg = ot.LJSPEECH
    m = TransformerTTS(cfg["idim"], cfg["odim"], device=dev, **{k: v for k, v in cfg.items() if k not in ("idim", "odim")})
    m.set_state_dict(ot.synth_params(12, cfg))
    step = TransformerTTSTrainStep(m, learning_rate=1e-3, guided_attn_loss_lambda=10.0)
    batch = workload(cfg, dev)
    B, T = batch["text"].shape
    L = batch["speech"].shape[1]
    for _ in range(3):                                              # eager, capture, replay
        losses = step.step(batch)
    torch.cuda.synchronize()
    assert step._graphs.replays >= 1, "the step did not replay as a CUDA graph"
    frames = int(batch["speech_lengths"].sum())
    flop = 3 * algorithmic_flop(cfg, B, T + 1, L)
    print(f"B={B} T={T + 1} L={L}: {frames} unpadded mel frames; loss {losses['loss'].item():.4f}; "
          f"peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                step.step(batch)
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=30, max_name_column_width=60)
        with open(os.path.join(args.profile, "transformer_tts_train_profile.txt"), "w") as f:
            f.write(f"card: {card()}\n3 steps, B={B} T={T + 1} L={L}\n{table}\n")
        print(table)
        return

    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rep in range(args.repeats):
        start.record()
        for _ in range(args.steps):
            step.step(batch)
        stop.record()
        torch.cuda.synchronize()
        ms = start.elapsed_time(stop) / args.steps
        print(f"repeat {rep}: {ms:.1f} ms per step over {args.steps} steps, {frames / (ms * 1e-3) / 1e3:.1f} k mel frames/s, "
              f"{flop / (ms * 1e-3) / 1e12:.1f} algorithmic TFLOP/s (3 x forward GEMM FLOP)")


if __name__ == "__main__":
    main()
