"""Time one WaveFlow training step (WaveFlowTrainStep.step: forward + WaveFlowLoss + backward replayed as one CUDA graph, then
Adam) with CUDA events on the reference's training batch (examples/waveflow/config.py: batch 8, clip_frames 65, hop 256 ->
audio (8, 16640), mel (8, 80, 65)), shipped model shape (8 flows x 8 layers, n_group 16), at 128 and 64 channels.

Algorithmic FLOP per step: 3 x the forward's n_flows * n_layers * B * (n_group - 1) * W * (40 C^2 + 4 C n_mels) (forward, data
gradient, weight gradient), reported against the 989 TFLOP/s dense-BF16 figure of the H100 SXM data sheet.

    python scripts/time_waveflow_train.py [--iters 10]
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DATASHEET_BF16_TFLOPS = 989.0
WORKLOADS = [("train batch", 8, 65, 128), ("train batch", 8, 65, 64)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not readable"
    return f"{name}, {q}"


def algorithmic_flop(m, batch, width):
    C = m.channels
    return 3 * m.n_flows * m.n_layers * batch * (m.n_group - 1) * width * (40 * C * C + 4 * C * m.n_mels)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU and has no CPU fallback")
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    for name, batch, frames, channels in WORKLOADS:
        m = ConditionalWaveFlow([16, 16], 8, 8, 16, channels, 80, (3, 3), device=dev)
        m.set_state_dict(owf.synth_params(5 if channels == 128 else 4, channels=channels))
        step = WaveFlowTrainStep(m)
        g = torch.Generator().manual_seed(7)
        mel = (torch.randn(batch, 80, frames, generator=g) * 0.5 - 3).to(dev)
        audio = ((torch.rand(batch, frames * 256, generator=g) * 2 - 1) * 0.5).to(dev)
        for _ in range(3):                                   # eager, capture, replay
            loss = step.step((mel, audio))
        torch.cuda.synchronize()
        assert step._graphs.replays >= 1, "the step did not replay as a CUDA graph"
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.iters):
            loss = step.step((mel, audio))
        stop.record()
        torch.cuda.synchronize()
        ms = start.elapsed_time(stop) / args.iters
        width = audio.shape[1] // 16
        tflops = algorithmic_flop(m, batch, width) / (ms * 1e-3) / 1e12
        print(f"{name}: B={batch} frames={frames} channels={channels} audio={tuple(audio.shape)}: {ms:.2f} ms per training step, "
              f"{batch * audio.shape[1] / (ms * 1e-3) / 1e3:.1f} k audio samples/s, {tflops:.1f} algorithmic TFLOP/s = "
              f"{100 * tflops / DATASHEET_BF16_TFLOPS:.1f} % of the 989 TFLOP/s dense-BF16 data-sheet peak "
              f"(loss {float(loss):.4f}, peak memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB)")
        del step, m
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()


if __name__ == "__main__":
    main()
