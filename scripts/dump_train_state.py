"""Fingerprint the training steps, to compare two builds of this repository bit for bit.

For each step class the small seeded model and batch of its GPU test run three `step` calls with CUDA graphs (eager, capture,
replay) and three without (PK_TRAIN_GRAPH=0, PK_CUDA_GRAPHS=0).  Per class and mode the JSON holds the SHA-256 of the flat
parameters, the flat gradient and both Adam moment buffers after the last step, the loss values of every step, and - eager mode -
the kernel launches of every step (`pk_launch_count`).  The FastSpeech2 and Parallel WaveGAN backward passes accumulate with
atomicAdd, so run a build twice before reading a difference between two builds as a change.

    python scripts/dump_train_state.py OUT_DIR [--name train_state.json]
"""
import argparse
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STEPS = 3


def sha(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def state(opt):
    """opt: a FlatAdam (its flat / gflat buffers and moments m / v)."""
    return dict(flat=sha(opt.flat), gflat=sha(opt.gflat), adam_m=sha(opt.m), adam_v=sha(opt.v))


def run(make, dev):
    """make(dev) -> (one_step() -> list of loss floats, states() -> dict); three steps with launch counts."""
    from parakeet_b200 import _lib
    one_step, states = make(dev)
    losses, launches = [], []
    for _ in range(STEPS):
        n0 = _lib.launch_count()
        out = one_step()
        torch.cuda.synchronize()
        launches.append(_lib.launch_count() - n0)
        losses.append(out)
    return dict(losses=losses, launches=launches, **states())


def fastspeech2(dev):
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2
    from parakeet_b200.training import FastSpeech2TrainStep
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, stop_gradient_from_pitch_predictor=True, device=dev)
    m.set_state_dict(ofs.synth_params(1))
    batch = ofs.synth_train_batch(5, [9, 14, 11], dur_range=(1, 4))
    ts = FastSpeech2TrainStep(m, learning_rate=1e-3, dropout=True, seed=3)
    return (lambda: [float(v) for v in ts.step(batch)]), (lambda: {"net": state(ts.opt)})


def waveflow(dev):
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    from parakeet_b200.training import WaveFlowTrainStep
    m = ConditionalWaveFlow([16, 16], 2, 3, 16, 64, 80, (3, 3), device=dev)
    m.set_state_dict(owf.synth_params(9, upsample_factors=(16, 16), n_flows=2, n_layers=3, n_group=16, channels=64, n_mels=80))
    g = torch.Generator().manual_seed(16)
    mel = (torch.randn(3, 80, 12, generator=g) * 0.5 - 3).to(dev)
    audio = ((torch.rand(3, 12 * 256 - 7, generator=g) * 2 - 1) * 0.5).to(dev)
    ts = WaveFlowTrainStep(m, learning_rate=2e-4)
    return (lambda: [float(ts.step((mel, audio)))]), (lambda: {"net": state(ts.opt)})


def speedyspeech(dev):
    from oracle import speedyspeech as oss
    from oracle import speedyspeech_train as sst
    from parakeet_b200.models import SpeedySpeech
    from parakeet_b200.training import SpeedySpeechTrainStep
    cfg = oss.SMALL_CFG
    m = SpeedySpeech(vocab_size=40, tone_size=None, device=dev, **cfg)
    m.set_state_dict(oss.synth_params(40, cfg))
    batch = {k: v.to(dev) for k, v in sst.synth_batch(50, [9, 6, 8]).items()}
    ts = SpeedySpeechTrainStep(m, max_grad_norm=1.0, learning_rate=2e-5)
    return (lambda: [float(v) for v in ts.step(batch).values()]), (lambda: {"net": state(ts.opt)})


def transformer_tts(dev):
    from oracle import transformer_tts_train as ot
    from parakeet_b200.models import TransformerTTS
    from parakeet_b200.training import TransformerTTSTrainStep
    cfg = ot.TRAIN_SMALL
    m = TransformerTTS(cfg["idim"], cfg["odim"], device=dev, **{k: v for k, v in cfg.items() if k not in ("idim", "odim")})
    m.set_state_dict(ot.synth_params(51, cfg))
    text, tl, sp, sl = ot.golden_batch(cfg, 52, lens=(9, 4, 6), frames=(40, 23, 31))
    batch = dict(text=text.to(dev), text_lengths=tl.to(dev), speech=sp.to(dev), speech_lengths=sl.to(dev))
    rates = {k: 0.1 for k in m.dropout_rates}
    ts = TransformerTTSTrainStep(m, learning_rate=1e-4, guided_attn_loss_lambda=10.0, dropout=rates, seed=9)
    return (lambda: [float(v) for v in ts.step(batch).values()]), (lambda: {"net": state(ts.opt)})


def ge2e(dev):
    """Three batch shapes A, B, A: the second A is captured while B's planes and graph are kept."""
    from oracle import ge2e as og
    from parakeet_b200.models import LSTMSpeakerEncoder
    from parakeet_b200.training import GE2ETrainStep
    cfg = (40, 3, 256, 256)
    m = LSTMSpeakerEncoder(*cfg, device=dev)
    m.set_state_dict(og.synth_params(13, *cfg))
    xs = [og.synth_utterances(30 + i, 20, t, 40).to(dev) for i, t in enumerate((50, 31, 50))]
    ts = GE2ETrainStep(m, num_speakers=4)
    it = iter(xs)
    return (lambda: [float(ts.step(next(it)))]), (lambda: {"net": state(ts.opt)})


def pwg(dev):
    from oracle import pwg as opwg
    from parakeet_b200.models import PWGDiscriminator, PWGGenerator
    from parakeet_b200.training import PWGTrainStep
    gen = PWGGenerator(**opwg.DEFAULT_GENERATOR_PARAMS, device=dev)
    gen.set_state_dict(opwg.synth_params(2, weight_norm=True))
    dis = PWGDiscriminator(device=dev, seed=6)
    noise, mel = opwg.synth_inputs(7, batch=2, mel_frames=20)
    wav = torch.randn(2, 1, 20 * 300, generator=torch.Generator().manual_seed(8)) * 0.3
    ts = PWGTrainStep(gen, dis, discriminator_train_start_steps=0)
    ts.iteration = 1                                         # past the start: generator (adversarial) and discriminator halves
    noise = noise.to(dev)

    def one_step():
        out = ts.update_core((wav, mel), noise=noise)
        return [float(out["generator_loss"]), float(out["discriminator_loss"])]
    return one_step, (lambda: {"generator": state(ts.g.opt), "discriminator": state(ts.d.opt)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--name", default="train_state.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the training steps have no CPU fallback")
    dev = torch.device("cuda:0")
    result = {"card": torch.cuda.get_device_name(0)}
    for mode, flag in (("graphs", "1"), ("eager", "0")):
        os.environ["PK_TRAIN_GRAPH"] = os.environ["PK_CUDA_GRAPHS"] = flag      # read when a step is constructed
        for name, make in (("FastSpeech2TrainStep", fastspeech2), ("WaveFlowTrainStep", waveflow), ("SpeedySpeechTrainStep", speedyspeech),
                           ("TransformerTTSTrainStep", transformer_tts), ("GE2ETrainStep", ge2e), ("PWGTrainStep", pwg)):
            result.setdefault(name, {})[mode] = run(make, dev)
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, args.name)
    with open(path, "w") as f:
        json.dump(result, f, indent=1, sort_keys=True)
    print(path)


if __name__ == "__main__":
    main()
