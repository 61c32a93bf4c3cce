"""cfg5: FastSpeech2 training step (forward + backward + NCCL gradient all-reduce + Adam), 8 utterances per GPU.
   python scripts/bench_train.py [--steps K]          or   torchrun --nproc-per-node N scripts/bench_train.py
   python scripts/bench_train.py --num-speakers 218   # the aishell3 model (spk_embed_dim 256, concat) at the same shape
Prints one JSON line from rank 0 (steps/s and mel-frames/s, whole job).  Run it with and without --num-speakers to see what
the speaker conditioning adds to the step."""
import argparse, json, math, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--per-gpu-batch", type=int, default=8)
ap.add_argument("--num-speakers", type=int, default=None, help="multi-speaker model (aishell3: 218, vctk: 109); default single speaker")
ap.add_argument("--spk-integration", choices=("concat", "add"), default="concat")
args = ap.parse_args()
rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)
from parakeet_b200.models import FastSpeech2
from parakeet_b200.training import FastSpeech2TrainStep
m = FastSpeech2(80, 80, adim=384, aheads=2, elayers=4, eunits=1536, dlayers=4, dunits=1536, positionwise_layer_type="conv1d",
                positionwise_conv_kernel_size=3, duration_predictor_layers=2, duration_predictor_chans=256, duration_predictor_kernel_size=3,
                postnet_layers=5, postnet_filts=5, postnet_chans=256, pitch_predictor_layers=5, pitch_predictor_chans=256,
                pitch_predictor_kernel_size=5, pitch_embed_kernel_size=1, energy_predictor_layers=2, energy_predictor_chans=256,
                energy_predictor_kernel_size=3, energy_embed_kernel_size=1, stop_gradient_from_pitch_predictor=True, device=dev, seed=1,  # same seed on every rank
                **(dict(num_speakers=args.num_speakers, spk_embed_dim=256, spk_embed_integration_type=args.spk_integration)
                   if args.num_speakers else {}))
ts = FastSpeech2TrainStep(m, learning_rate=1e-3, dropout=False)
g = torch.Generator().manual_seed(5 + rank)              # every rank gets its own shard of the (synthetic) data
B = args.per_gpu_batch
lengths = torch.randint(60, 141, (B,), generator=g).tolist()
Tm = max(lengths)
text = torch.zeros(B, Tm, dtype=torch.int64); ds = torch.zeros(B, Tm, dtype=torch.int64)
ps = torch.zeros(B, Tm, 1); es = torch.zeros(B, Tm, 1)
for i, n in enumerate(lengths):
    text[i, :n] = torch.randint(1, 79, (n,), generator=g); ds[i, :n] = torch.randint(2, 13, (n,), generator=g)
    ps[i, :n] = torch.randn(n, 1, generator=g); es[i, :n] = torch.randn(n, 1, generator=g)
olens = ds.sum(1); Lm = int(olens.max())
ys = torch.zeros(B, Lm, 80)
for i in range(B):
    ys[i, :int(olens[i])] = torch.randn(int(olens[i]), 80, generator=g)
batch = dict(text=text, text_lengths=torch.tensor(lengths), speech=ys, speech_lengths=olens, durations=ds, pitch=ps, energy=es)
if args.num_speakers:
    batch["spk_id"] = torch.randint(0, args.num_speakers, (B,), generator=torch.Generator().manual_seed(7 + rank))
batch = {k: v.to(dev) for k, v in batch.items()}
for _ in range(args.warmup):
    l = ts.step(batch)
if world > 1: dist.barrier()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(args.steps):
    l = ts.step(batch)
e1.record()
if world > 1: dist.barrier()
torch.cuda.synchronize()
ms = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
frames = torch.tensor([float(olens.sum())], device=dev, dtype=torch.float64)
if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX); dist.all_reduce(frames)
if rank == 0:
    per = float(ms) / args.steps
    print(json.dumps({"workload": "fastspeech2_train_step", "n_gpus": world, "global_batch": B * world, "ms_per_step": per,
                      "steps_per_s": 1e3 / per, "mel_frames_per_s": float(frames) / per * 1e3, "loss": [float(v) for v in l],
                      "grad_allreduce_mb": ts.gflat.numel() * 4 / 1e6, "num_speakers": args.num_speakers,
                      "spk_integration": args.spk_integration if args.num_speakers else None}))
if world > 1: dist.destroy_process_group()
