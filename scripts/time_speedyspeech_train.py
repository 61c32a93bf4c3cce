"""Time SpeedySpeechTrainStep.step (the baker recipe's acoustic model, examples/speedyspeech/baker/conf/default.yaml: batch 64,
hidden 128, kernel 3, 10 encoder and 18 decoder residual blocks, Adam 2e-3 with ClipGradByGlobalNorm(1)) with CUDA events
around CUDA-graph replays, after the timed shape has been warmed up (eager, capture, replay).

Workload: 64 utterances of T ~ U{60..140} phonemes with tones, durations U{2..8} frames per phoneme (about 5, as
scripts/time_speedyspeech.py's duration head gives), seeded weights.  Algorithmic TFLOP/s counts 3 x the forward's Conv1D /
Linear FLOP over ALL B * T and B * L rows (padded rows are live in training), 2 FLOP per multiply-add, one pass.

    python scripts/time_speedyspeech_train.py [--steps 20] [--repeats 2] [--profile DIR]

--profile (a separate run: tracing slows the host) writes torch.profiler's kernel table of 3 steps to DIR.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

BATCH, T_MIN, T_MAX, TONES = 64, 60, 140, 6


def workload(dev):
    g = torch.Generator().manual_seed(2021)
    lengths = torch.randint(T_MIN, T_MAX + 1, (BATCH,), generator=g)
    T = int(lengths.max())
    phones, tones, dur = (torch.zeros(BATCH, T, dtype=torch.int64) for _ in range(3))
    for i, n in enumerate(lengths.tolist()):
        phones[i, :n] = torch.randint(1, 40, (n,), generator=g)
        tones[i, :n] = torch.randint(1, TONES, (n,), generator=g)
        dur[i, :n] = torch.randint(2, 9, (n,), generator=g)
    frames = dur.sum(1)
    feats = torch.randn(BATCH, int(frames.max()), 80, generator=g)
    feats[torch.arange(feats.shape[1])[None, :] >= frames[:, None]] = 0
    batch = dict(phones=phones, tones=tones, num_phones=lengths, num_frames=frames, feats=feats, durations=dur)
    return {k: v.to(dev) for k, v in batch.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--profile", default=None, help="directory for the torch.profiler table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU and has no CPU fallback")
    from time_speedyspeech import algorithmic_flop, card
    from oracle import speedyspeech as oss
    from parakeet_b200.models import SpeedySpeech
    from parakeet_b200.training import SpeedySpeechTrainStep
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    cfg = oss.SHIPPED_CFG
    m = SpeedySpeech(40, tone_size=TONES, device=dev, **cfg)
    m.set_state_dict(oss.synth_params(3, cfg, tone_size=TONES))
    step = SpeedySpeechTrainStep(m, check_durations=False)          # no device->host copy in the timed loop
    batch = workload(dev)
    B, T = batch["phones"].shape
    L = batch["feats"].shape[1]
    for _ in range(3):                                              # eager, capture, replay
        losses = step.step(batch)
    torch.cuda.synchronize()
    assert step._graphs.replays >= 1, "the step did not replay as a CUDA graph"
    frames = int(batch["num_frames"].sum())
    flop = 3 * B * algorithmic_flop(cfg, T, L)
    print(f"B={B} T={T} L={L}: {B * T} token rows, {B * L} frame rows ({frames} unpadded mel frames); loss {losses['loss'].item():.4f}; "
          f"peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                step.step(batch)
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=30, max_name_column_width=60)
        with open(os.path.join(args.profile, "speedyspeech_train_profile.txt"), "w") as f:
            f.write(f"card: {card()}\n3 steps, B={B} T={T} L={L}\n{table}\n")
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
        print(f"repeat {rep}: {ms:.2f} ms per step over {args.steps} steps, {frames / (ms * 1e-3) / 1e6:.3f} M mel frames/s, "
              f"{flop / (ms * 1e-3) / 1e12:.1f} algorithmic TFLOP/s (3 x forward Conv1D / Linear FLOP)")


if __name__ == "__main__":
    main()
