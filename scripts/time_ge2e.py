"""Time the GE2E speaker encoder on the GPU (CUDA events, graph replay for the training step):
  - GE2ETrainStep at the recipe shape (64 speakers x 10 utterances x 160 frames x 40 mels, 3 LSTM layers x 256);
  - LSTMSpeakerEncoder.embed_utterances over a few thousand 160-frame partials;
  - for context, torch's cuDNN nn.LSTM forward on the same shapes and card.
Prints the card's name and power limit and algorithmic FLOP/s from shapes: per row-step per layer 2 * 4H * (I + H) for the forward,
3x that for the training step.

    python scripts/time_ge2e.py [--steps 20] [--partials 4096]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "nvidia-smi unavailable"
    return f"{torch.cuda.get_device_name(0)} ({q})"


def timed(fn, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def flops_fwd(rows, T, layers, I, H):
    return sum(2 * 4 * H * ((I if l == 0 else H) + H) for l in range(layers)) * rows * T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--partials", type=int, default=4096)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA GPU")
    from parakeet_b200.models import LSTMSpeakerEncoder
    from parakeet_b200.training import GE2ETrainStep
    dev = torch.device("cuda:0")
    print("card:", card())
    N, M, T, I, H, L = 64, 10, 160, 40, 256, 3
    torch.manual_seed(0)
    m = LSTMSpeakerEncoder(I, L, H, H, device=dev)
    step = GE2ETrainStep(m, num_speakers=N)
    specs = torch.randn(N * M, T, I, device=dev) * 0.5
    for _ in range(3):
        step.step(specs)
    ms = timed(lambda: step.step(specs), a.steps)
    f = 3 * flops_fwd(N * M, T, L, I, H)
    print(f"train step {N}x{M}x{T}x{I}, {L}x{H}: {ms:.3f} ms/step, {f / ms / 1e9:.2f} TFLOP/s algorithmic")
    parts = [torch.randn(a.partials, T, I, device=dev) * 0.5]
    with torch.no_grad():
        m.embed_utterances(parts)
        ms_e = timed(lambda: m.embed_utterances(parts), 5)
    f = flops_fwd(a.partials, T, L, I, H)
    print(f"embed_utterances {a.partials} partials x {T}: {ms_e:.3f} ms, {f / ms_e / 1e9:.2f} TFLOP/s algorithmic")
    torch.backends.cudnn.allow_tf32 = False             # the context number is cuDNN in full fp32, like the kernels' bf16x3
    ref = torch.nn.LSTM(I, H, L, batch_first=True).to(dev)
    for rows, what in ((N * M, "recipe batch"), (a.partials, "partials")):
        x = torch.randn(rows, T, I, device=dev)
        with torch.no_grad():
            ref(x)
            ms_c = timed(lambda: ref(x), 10)
        print(f"torch cuDNN nn.LSTM forward ({what}, {rows} x {T}, fp32): {ms_c:.3f} ms, "
              f"{flops_fwd(rows, T, L, I, H) / ms_c / 1e9:.2f} TFLOP/s algorithmic")


if __name__ == "__main__":
    main()
