#!/usr/bin/env python
"""Where the time of the Parallel WaveGAN generator forward (bench.py's workload: batch 32, 80-mel x 400 frames, 3.84 M
samples per step) goes, and A/B runs of bench.py across source trees.

  python scripts/prof_pwg.py [--out DIR] [--steps N]
      torch.profiler per-kernel table of the forward (name, launches, total ms) -> DIR/kernels.txt, then the residual-layer
      kernel's average time (CUDA events around the 30 launches, no profiler) with its HBM and tensor shares, and the card's
      name, power limit and SM clock.

  python scripts/prof_pwg.py --compare TREE [TREE ...] [--rounds R] [--out DIR]
      runs `bench.py --no-extra --dump-outputs` of each tree (each built in place), alternating, R >= 3 rounds; reports the
      median and spread of `value` and `roofline.launch_ms` per tree and whether every dumped waveform equals the first
      tree's bit for bit.

Shares: HBM = 1 024 B/sample per layer (x read 256, y write 256, skip read-modify-write 512) over the layer time, against
3.35 TB/s; tensor = 208 896 executed FLOP/sample per layer over the layer time (51 wgmma m64n128k16 per 64 rows: GEMM1 3 taps x 4 K-steps + 1 conditioning K-step, GEMM2 4 K-steps,
split-bf16, 3 passes each), against 989 TFLOP/s (data-sheet dense bf16 at 700 W; a card with a lower power limit clocks lower).
Both are a middle layer's: the layer time is the mean over the 30 launches, and the first layer (no x read, a skip store: 512 B/sample,
15 wgmma per 64 rows) and the last (no skip write, the tail on top: 768 B/sample) move less, so the shares slightly understate a middle layer's.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BATCH, FRAMES, HOP, LAYERS = 32, 400, 300, 30
SAMPLES = BATCH * FRAMES * HOP
HBM_BYTES_PER_SAMPLE = 1024
TENSOR_FLOP_PER_SAMPLE = 51 * 2 * 64 * 128 * 16 // 64          # 208 896
HBM_PEAK_GBS, BF16_PEAK_TFLOPS = 3350.0, 989.0
LAYER_KERNEL = "pwg_layer_fc_kernel"


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=20)
        f = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), f))
    except Exception as ex:
        return {"error": repr(ex)}


def shares(layer_ms):
    s = layer_ms * 1e-3
    return {"layer_ms": layer_ms,
            "hbm_gbs": SAMPLES * HBM_BYTES_PER_SAMPLE / s / 1e9,
            "hbm_share": SAMPLES * HBM_BYTES_PER_SAMPLE / s / 1e9 / HBM_PEAK_GBS,
            "tensor_tflops": SAMPLES * TENSOR_FLOP_PER_SAMPLE / s / 1e12,
            "tensor_share": SAMPLES * TENSOR_FLOP_PER_SAMPLE / s / 1e12 / BF16_PEAK_TFLOPS}


def profile(args):
    sys.path.insert(0, ROOT)
    import torch
    from parakeet_b200.models import PWGGenerator
    if not torch.cuda.is_available():
        raise SystemExit("prof_pwg.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    gen = PWGGenerator(layers=LAYERS, stacks=3, residual_channels=64, gate_channels=128, skip_channels=64, aux_channels=80,
                       aux_context_window=2, upsample_scales=[4, 5, 3, 5], use_weight_norm=True, device=dev, seed=2)
    gen.remove_weight_norm()
    g = torch.Generator().manual_seed(1002)                     # bench.py's inputs
    c = torch.randn(BATCH, 80, FRAMES, generator=g)
    c = torch.cat([c[:, :, :1].expand(-1, -1, 2), c, c[:, :, -1:].expand(-1, -1, 2)], dim=-1).contiguous().to(dev)
    x = torch.randn(BATCH, 1, FRAMES * HOP, generator=g).to(dev)
    gen._layer_events = []                                      # eager launches: one profiler row per kernel launch
    for _ in range(3):
        gen(x, c)
    torch.cuda.synchronize()

    # residual-layer time from CUDA events around the 30 launches, profiler off
    gen._layer_events = []
    for _ in range(args.steps):
        gen(x, c)
    torch.cuda.synchronize()
    per_step = [a.elapsed_time(b) for a, b in gen._layer_events]
    layer_ms = statistics.median(per_step) / LAYERS

    from torch.profiler import ProfilerActivity, profile as tprofile
    gen._layer_events = []
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.prof_steps):
            gen(x, c)
        torch.cuda.synchronize()
    gen._layer_events = None
    rows = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        r = rows.setdefault(e.name, [0, 0.0])
        r[0] += 1
        r[1] += e.device_time_total / 1e3
    table = sorted(((n, k / args.prof_steps, ms / args.prof_steps) for n, (k, ms) in rows.items()), key=lambda r: -r[2])
    total = sum(r[2] for r in table)
    info = gpu_info()
    os.makedirs(args.out, exist_ok=True)
    lines = [f"per-kernel device time of one forward (batch {BATCH} x {FRAMES} frames, {SAMPLES} samples), "
             f"mean of {args.prof_steps} profiled steps; {info}",
             f"{'kernel':<90} {'launches':>9} {'total ms':>10} {'share':>7}"]
    for n, k, ms in table:
        lines.append(f"{n[:90]:<90} {k:>9.0f} {ms:>10.3f} {ms / total:>7.1%}")
    lines.append(f"{'sum':<90} {sum(r[1] for r in table):>9.0f} {total:>10.3f}")
    text = "\n".join(lines)
    with open(os.path.join(args.out, "kernels.txt"), "w") as f:
        f.write(text + "\n")
    print(text)
    prof_layer = [ms / k for n, k, ms in table if LAYER_KERNEL in n and k]
    res = {"gpu": info, "events_layer": shares(layer_ms), "events_step_layers_ms": per_step,
           "profiler_layer_ms": prof_layer[0] if prof_layer else None, "profiler_forward_ms": total}
    with open(os.path.join(args.out, "layer.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


def compare(args):
    trees = [os.path.abspath(t) for t in args.compare]
    args.out = os.path.abspath(args.out)
    os.makedirs(args.out, exist_ok=True)
    runs = {t: [] for t in trees}
    for r in range(max(args.rounds, 3)):
        for i, t in enumerate(trees):
            dump = os.path.join(args.out, f"tree{i}_round{r}")
            cmd = [sys.executable, os.path.join(t, "bench.py"), "--no-extra", "--gpus", "1", "--steps", str(args.steps),
                   "--warmup", "3", "--dump-outputs", dump]
            p = subprocess.run(cmd, cwd=t, capture_output=True, text=True)
            line = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
            if p.returncode or not line:
                print(f"[{t}] round {r} failed ({p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}", flush=True)
                raise SystemExit(1)
            j = json.loads(line[-1])
            runs[t].append({"value": j["value"], "launch_ms": j["roofline"]["launch_ms"], "sm_mhz": j["clocks"]["sm_mhz"],
                            "dump": os.path.join(dump, "pwg_wav.npy")})
            print(f"round {r} tree{i} value {j['value'] / 1e6:.2f} M samples/s, layer {j['roofline']['launch_ms']:.3f} ms, "
                  f"SM {j['clocks']['sm_mhz']} MHz", flush=True)
    import numpy as np
    ref = np.load(runs[trees[0]][0]["dump"])
    out = {"gpu": gpu_info(), "trees": []}
    for i, t in enumerate(trees):
        v = [x["value"] for x in runs[t]]
        lm = [x["launch_ms"] for x in runs[t]]
        same = all(np.array_equal(np.load(x["dump"]).view(np.uint32), ref.view(np.uint32)) for x in runs[t])
        maxdiff = max(float(np.abs(np.load(x["dump"]).astype(np.float64) - ref).max()) for x in runs[t])
        rec = {"tree": t, "value_median": statistics.median(v), "value_min": min(v), "value_max": max(v),
               "launch_ms_median": statistics.median(lm), "launch_ms_min": min(lm), "launch_ms_max": max(lm),
               "bit_identical_to_tree0": same, "max_abs_diff_to_tree0": maxdiff,
               "layer_shares": shares(statistics.median(lm)), "runs": runs[t]}
        out["trees"].append(rec)
        print(f"tree{i} {t}: value median {rec['value_median'] / 1e6:.2f} M/s [{min(v) / 1e6:.2f}, {max(v) / 1e6:.2f}], "
              f"layer median {rec['launch_ms_median']:.3f} ms [{min(lm):.3f}, {max(lm):.3f}], bit-identical {same}, "
              f"max |diff| {maxdiff:.3g}, HBM share {rec['layer_shares']['hbm_share']:.1%}, "
              f"tensor share {rec['layer_shares']['tensor_share']:.1%}", flush=True)
    for t in trees:                                              # 15 MB each: keep the verdict, not the waveforms
        for x in runs[t]:
            os.remove(x["dump"])
            os.rmdir(os.path.dirname(x["dump"]))
            del x["dump"]
    base = out["trees"][0]["value_median"]
    for rec in out["trees"][1:]:
        rec["speedup_vs_tree0"] = rec["value_median"] / base
        print(f"{rec['tree']}: {rec['speedup_vs_tree0']:.3f}x tree0")
    print(json.dumps(out["gpu"]))
    with open(os.path.join(args.out, "compare.json"), "w") as f:
        json.dump(out, f, indent=1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=os.path.join(ROOT, "build", "prof_pwg"))
    ap.add_argument("--steps", type=int, default=20, help="timed forwards (events; bench steps with --compare)")
    ap.add_argument("--prof-steps", type=int, default=3, help="profiled forwards")
    ap.add_argument("--compare", nargs="+", metavar="TREE", help="source trees to A/B with bench.py (the first is the reference)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    compare(args) if args.compare else profile(args)


if __name__ == "__main__":
    main()
