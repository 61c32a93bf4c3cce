"""Time Tacotron2 on the GPU with CUDA events (every shape warmed up first):
  - infer at B = 1 for the ljspeech and aishell3 configs, T_enc = 150, exactly N decoder steps (stop token with a bias of -1e4);
    reports us per decoder step, mel frames/s, the real-time factor at hop 256 / 22 050 Hz, weight bytes per step and the implied
    bandwidth against the 3.35 TB/s data sheet;
  - the teacher-forced forward at the validation batch (32 utterances, T_mel up to 800);
  - one extra run of the ljspeech infer with the decoder's phase timers: per phase, the time between the hand-offs that enclose
    it and the hand-off's own latency (the shortest wait of any CTA from its arrival to the release);
  - for context, the eager fp32 oracle decoder (torch, TF32 off) on the same card for a few steps, with the prenet dropout at 0
    so that no host-side mask generation is timed;
  - with --e2e, the aishell3 voice-cloning chain (GE2E embedding -> Tacotron2.infer -> 128-channel WaveFlow), seconds of audio
    per second.
Prints the card's name, power limit and max SM clock in the same run.

    python scripts/time_tacotron2.py [--steps 800] [--e2e]
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.time_ge2e import card, timed  # noqa: E402

HOP, SR, HBM = 256, 22050, 3.35e12


def weight_bytes(cfg):
    """fp32 weights the decoder reads per step (prenet, both LSTMCells, query layer, projection, stop)."""
    dk = cfg["d_encoder"] + (cfg["d_global_condition"] or 0)
    dm = cfg["d_mels"] * cfg["reduction_factor"]
    n = dm * 256 + 256 * 256 + 4096 * (256 + dk + 1024) + 4096 * (1024 + dk + 1024) + 1024 * 128 + (1024 + dk) * (dm + 1)
    return 4 * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=800)
    ap.add_argument("--t-enc", type=int, default=150)
    ap.add_argument("--e2e", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA GPU")
    import oracle.tacotron2 as ot
    from parakeet_b200 import _lib, ops
    from parakeet_b200.models import Tacotron2
    dev = torch.device("cuda:0")
    print(card())
    for name, base in (("ljspeech", ot.LJSPEECH), ("aishell3", ot.AISHELL3)):
        cfg = dict(base, use_stop_token=True)
        p = ot.synth_params(0, cfg, stop_bias=-1e4)
        m = Tacotron2(device=dev, **cfg)
        m.set_state_dict(p)
        text, tones = ot.synth_text(1, 1, a.t_enc, cfg["vocab_size"], cfg["n_tones"])
        gc = torch.randn(1, 256, device=dev) if cfg["d_global_condition"] else None
        kw = dict(tones=tones.to(dev) if tones is not None else None, global_condition=gc, seed=1)
        run = lambda: m.infer(text.to(dev), max_decoder_steps=a.steps, **kw)
        assert run()["mel_output"].shape[1] == a.steps
        ms = timed(run, 3)
        us = ms * 1e3 / a.steps
        wb = weight_bytes(cfg)
        print(f"{name} infer B=1 T_enc={a.t_enc} N={a.steps}: {ms:.1f} ms, {us:.1f} us/step, {a.steps / ms * 1e3:.0f} frames/s, "
              f"RTF {ms / 1e3 / (a.steps * HOP / SR):.3f}, {wb / 1e6:.1f} MB weights/step -> {wb / (us * 1e-6) / 1e9:.0f} GB/s "
              f"({wb / (us * 1e-6) / HBM * 100:.0f}% of 3.35 TB/s)")
        if name == "ljspeech":
            prof = torch.zeros(int(_lib.lib().pk_taco2_prof_len()), dtype=torch.int64, device=dev)
            keys, pkeys = m._encode(text.to(dev), None, None, None)
            ops.taco2_decode(m._packs()["dec"], keys, pkeys, a.steps, teacher=False, p_prenet=0.5, seed=1, prof=prof)
            torch.cuda.synchronize()
            pr = prof.reshape(-1, 2, 6)[:torch.count_nonzero(prof.reshape(-1, 12).sum(1))].double() / a.steps / 1e3
            names = ("prenet 1", "prenet 2", "attention LSTMCell", "attention", "decoder LSTMCell", "projection + stop")
            print("  phase timers (us per step): " + "; ".join(f"{n} {pr[0, 0, i]:.1f} (hand-off {pr[:, 1, i].min():.1f})"
                                                            for i, n in enumerate(names)))
        # validation batch: 32 utterances, ragged text, T_mel 800
        B, T_mel = 32, 800
        tb, tnb = ot.synth_text(2, B, a.t_enc, cfg["vocab_size"], cfg["n_tones"])
        lens = torch.randint(a.t_enc // 2, a.t_enc + 1, (B,))
        lens[0] = a.t_enc
        mels = torch.randn(B, T_mel, 80, device=dev)
        gcb = torch.randn(B, 256, device=dev) if cfg["d_global_condition"] else None
        fwd = lambda: m.forward(tb.to(dev), lens.to(dev), mels, torch.full((B,), T_mel, device=dev),
                                tones=tnb.to(dev) if tnb is not None else None, global_condition=gcb, seed=1)
        fwd()
        ms = timed(fwd, 2)
        print(f"{name} forward B={B} T_mel={T_mel}: {ms:.1f} ms, {ms * 1e3 / T_mel:.1f} us/step")
        # eager fp32 oracle on the same card, a few steps
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        pd = {k: v.to(dev) for k, v in p.items()}
        cfg0 = dict(cfg, p_prenet_dropout=0.0)
        keys = torch.randn(1, a.t_enc, 512 + (cfg["d_global_condition"] or 0), device=dev)
        n_or = 50
        ot.decode(pd, cfg0, keys, max_decoder_steps=5, seed=1, dtype=torch.float32)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ot.decode(pd, cfg0, keys, max_decoder_steps=n_or, seed=1, dtype=torch.float32)
        torch.cuda.synchronize()
        print(f"{name} eager fp32 torch decoder (prenet dropout 0) on the same card: {(time.perf_counter() - t0) * 1e6 / n_or:.0f} us/step")
    if a.e2e:
        from parakeet_b200.models import ConditionalWaveFlow, LSTMSpeakerEncoder
        enc = LSTMSpeakerEncoder(40, 3, 256, 256, device=dev)
        voc = ConditionalWaveFlow([16, 16], 8, 8, 16, 128, 80, (3, 3), device=dev)
        cfg = dict(ot.AISHELL3, use_stop_token=True)
        m = Tacotron2(device=dev, **cfg)
        m.set_state_dict(ot.synth_params(0, cfg, stop_bias=-1e4))
        text, tones = ot.synth_text(3, 1, 60, cfg["vocab_size"], cfg["n_tones"])
        ref = torch.randn(3, 160, 40, device=dev)

        def chain():
            e = enc.embed_utterance(ref).reshape(1, 256)
            mel = m.infer(text.to(dev), max_decoder_steps=a.steps, tones=tones.to(dev), global_condition=e, seed=1)["mel_outputs_postnet"]
            return voc.infer(mel.transpose(1, 2).contiguous())
        wav = chain()
        ms = timed(chain, 2)
        sec = wav.shape[-1] / SR
        print(f"voice cloning chain ({a.steps} frames, {sec:.2f} s of audio): {ms:.1f} ms, {sec / (ms / 1e3):.1f} s of audio per s")


if __name__ == "__main__":
    main()
