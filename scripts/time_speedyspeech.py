"""Time SpeedySpeech.batch_inference (the baker recipe's acoustic model, examples/speedyspeech/baker) with CUDA events, as
CUDA-graph replays after every shape has been warmed up.

Workload: a synthetic baker-shaped batch - 32 utterances of T ~ U{60..140} phonemes with tones, the shipped config
(examples/speedyspeech/baker/conf/default.yaml: hidden 128, kernel 3, 10 encoder and 18 decoder residual blocks), seeded
weights whose duration head gives about 5 frames per phoneme.  Each call includes its one device->host copy (the frame counts).
Algorithmic FLOP per utterance (`algorithmic_flop`, 2 FLOP per multiply-add, one pass - the split-bf16 passes and the halo
rows the kernel also computes are not counted) is reported against the 989 TFLOP/s dense-BF16 figure of the H100 SXM data sheet.

    python scripts/time_speedyspeech.py [--iters 20] [--e2e] [--profile DIR]

--e2e chains SpeedySpeechInference -> PWGInference on the baker Parallel WaveGAN (24 kHz, hop 300, upsample [4, 5, 3, 5]),
utterance by utterance as the recipe's synthesize_e2e.py does, and reports audio samples/s.  --profile writes the per-kernel
torch.profiler table of batch_inference to DIR (a separate run: tracing slows the host).
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DATASHEET_BF16_TFLOPS = 989.0
BATCH, T_MIN, T_MAX, TONES = 32, 60, 140, 6


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not readable"
    return f"{name}, {q}"


def algorithmic_flop(cfg, t_phones, frames, odim=80):
    """Multiply-adds x 2 of one utterance: encoder (prenet, 2 convs per block, postnet1, postnet2), duration predictor
    (kernel 4, 3, 1 blocks and the Linear to 1), decoder (2 convs per block, postnet1, the postnet2 block, output Linear)."""
    C, ke, kd = cfg["encoder_hidden_size"], cfg["encoder_kernel_size"], cfg["decoder_kernel_size"]
    enc = t_phones * (3 * C * C + 2 * len(cfg["encoder_dilations"]) * ke * C * C)
    dur = t_phones * ((4 + 3 + 1) * C * C + C)
    dec = frames * ((2 * len(cfg["decoder_dilations"]) + 2) * kd * C * C + C * C + C * odim)
    return 2 * (enc + dur + dec)


def workload(dev):
    g = torch.Generator().manual_seed(2021)
    lengths = torch.randint(T_MIN, T_MAX + 1, (BATCH,), generator=g)
    text = torch.zeros(BATCH, T_MAX, dtype=torch.int64)
    tones = torch.zeros(BATCH, T_MAX, dtype=torch.int64)
    for i, n in enumerate(lengths.tolist()):
        text[i, :n] = torch.randint(1, 40, (n,), generator=g)
        tones[i, :n] = torch.randint(1, TONES, (n,), generator=g)
    return text.to(dev), lengths.to(dev), tones.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--e2e", action="store_true")
    ap.add_argument("--profile", default=None, help="directory for the torch.profiler table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU and has no CPU fallback")
    from oracle import speedyspeech as oss
    from parakeet_b200.models import SpeedySpeech
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    cfg = oss.SHIPPED_CFG
    m = SpeedySpeech(40, tone_size=TONES, device=dev, **cfg).eval()
    m.set_state_dict(oss.synth_params(3, cfg, tone_size=TONES))
    text, lengths, tones = workload(dev)
    for _ in range(3):                                       # eager, capture, replay
        mel, frames, _ = m.batch_inference(text, lengths, tones)
    torch.cuda.synchronize()
    assert m._graphs.replays >= 2, "batch_inference did not replay as CUDA graphs"
    n_frames = int(frames.sum())
    flop = sum(algorithmic_flop(cfg, int(t), int(f)) for t, f in zip(lengths.tolist(), frames.tolist()))

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                m.batch_inference(text, lengths, tones)
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
        with open(os.path.join(args.profile, "speedyspeech_profile.txt"), "w") as f:
            f.write(f"card: {card()}\n5 calls of batch_inference, B={BATCH}, {n_frames} mel frames per call\n{table}\n")
        print(table)
        return

    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.iters):
        mel, frames, _ = m.batch_inference(text, lengths, tones)
    stop.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(stop) / args.iters
    tflops = flop / (ms * 1e-3) / 1e12
    print(f"batch_inference: B={BATCH} phonemes={int(lengths.sum())} (T {T_MIN}..{T_MAX}) mel frames={n_frames} "
          f"(padded {tuple(mel.shape)}): {ms:.3f} ms per call, {n_frames / (ms * 1e-3) / 1e6:.3f} M mel frames/s, "
          f"{tflops:.1f} algorithmic TFLOP/s = {100 * tflops / DATASHEET_BF16_TFLOPS:.1f} % of the 989 TFLOP/s dense-BF16 "
          f"data-sheet peak")

    if args.e2e:
        from oracle import pwg as opwg
        from parakeet_b200.models import PWGGenerator, PWGInference, SpeedySpeechInference
        from parakeet_b200.modules.normalizer import ZScore
        gen = PWGGenerator(**opwg.DEFAULT_GENERATOR_PARAMS, device=dev)
        gen.set_state_dict(opwg.synth_params(2, weight_norm=True))
        gen.remove_weight_norm()
        g = torch.Generator().manual_seed(5)
        ss = SpeedySpeechInference(ZScore(torch.randn(80, generator=g) * 0.2, torch.rand(80, generator=g) + 0.5, device=dev), m)
        voc = PWGInference(ZScore(torch.randn(80, generator=g) * 0.2, torch.rand(80, generator=g) + 0.5, device=dev), gen)
        utts = [(text[i, :n], tones[i, :n]) for i, n in enumerate(lengths.tolist())]

        def run():
            return sum(voc(ss(t, tn)).shape[0] for t, tn in utts)
        for _ in range(2):
            samples = run()
        torch.cuda.synchronize()
        start.record()
        iters = max(1, args.iters // 4)
        for _ in range(iters):
            samples = run()
        stop.record()
        torch.cuda.synchronize()
        ms = start.elapsed_time(stop) / iters
        print(f"e2e SpeedySpeechInference -> PWGInference, {BATCH} utterances one at a time: {samples} samples "
              f"({samples / 24000:.1f} s of 24 kHz audio) in {ms:.1f} ms = {samples / (ms * 1e-3) / 1e6:.2f} M samples/s")


if __name__ == "__main__":
    main()
