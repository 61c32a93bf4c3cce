"""Tacotron2 restated in torch (fp32 or fp64) for the parity tests (reference: parakeet/models/tacotron2.py, modules/attention.py
LocationSensitiveAttention, modules/conv.py Conv1dBatchNorm, modules/losses.py guided_attention_loss).

Eval semantics: the encoder, attention, decoder and postnet dropouts are identity; the prenet dropout is always on (the
reference calls F.dropout(..., training=True)), drawn here with PhiloxDropout(seed, step = decoder step) at sites
PRENET_SITES on the (B, 256) activations, the convention of the CUDA decoder.  Keys are the reference's (Paddle 2.1)
state-dict keys; Linear weights are [in, out], Conv1D weights [out, in, k].
"""
import math

import numpy as np
import torch

from .fastspeech2 import PhiloxDropout

PRENET_SITES = (0, 1)
LSTM_PARTS = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")

# constructor defaults (tacotron2.py:600-623) and the two shipped recipes (examples/tacotron2/ljspeech, tacotron2_aishell3)
DEFAULTS = dict(d_mels=80, d_encoder=512, encoder_conv_layers=3, encoder_kernel_size=5, d_prenet=256, d_attention_rnn=1024,
                d_decoder_rnn=1024, attention_filters=32, attention_kernel_size=31, d_attention=128, d_postnet=512,
                postnet_kernel_size=5, postnet_conv_layers=5, reduction_factor=1, p_encoder_dropout=0.5, p_prenet_dropout=0.5,
                p_attention_dropout=0.1, p_decoder_dropout=0.1, p_postnet_dropout=0.5, n_tones=None, d_global_condition=None,
                use_stop_token=False)
LJSPEECH = dict(DEFAULTS, vocab_size=37)
AISHELL3 = dict(DEFAULTS, vocab_size=69, n_tones=10, d_global_condition=256)

# the reference-executed fixture (scripts/make_golden_ref.py tacotron2): (config, weight seed), all with p_prenet_dropout = 0
GOLDEN_CONFIGS = {
    "small": (dict(DEFAULTS, vocab_size=20, d_mels=8, d_postnet=32, postnet_conv_layers=3, encoder_conv_layers=2, use_stop_token=True,
                   p_prenet_dropout=0.0), 71),
    "ljspeech": (dict(LJSPEECH, p_prenet_dropout=0.0), 72),
    "aishell3": (dict(AISHELL3, p_prenet_dropout=0.0), 73),
}


def golden_inputs(cfg, seed):
    """The fixture's teacher-forced batch: 3 utterances of text (9, 6, 4 tokens), 10 mel frames, output_lens (10, 7, 5)."""
    g = torch.Generator().manual_seed(seed)
    B, T, T_mel = 3, 9, 10
    text = torch.randint(0, cfg["vocab_size"], (B, T), generator=g)
    tones = torch.randint(1, cfg["n_tones"], (B, T), generator=g) if cfg["n_tones"] else None
    gc = torch.randn(B, cfg["d_global_condition"], generator=g) if cfg["d_global_condition"] else None
    mels = torch.randn(B, T_mel, cfg["d_mels"], generator=g) - 1.0
    return dict(text=text, tones=tones, gc=gc, mels=mels, text_lens=torch.tensor([9, 6, 4]), output_lens=torch.tensor([10, 7, 5]))


def cfg_of(**kw):
    c = dict(DEFAULTS)
    c.update(kw)
    return c


def param_shapes(cfg):
    """{key: shape} of the reference module built with cfg (Paddle 2.1 names)."""
    c = cfg
    de, dm = c["d_encoder"], c["d_mels"] * c["reduction_factor"]
    dk = de + (c["d_global_condition"] or 0)
    s = {"embedding.weight": (c["vocab_size"], de)}
    if c["n_tones"]:
        s["embedding_tones.weight"] = (c["n_tones"], de)

    def conv_bn(prefix, cin, cout, k):
        s[prefix + "conv.weight"] = (cout, cin, k)
        s[prefix + "conv.bias"] = (cout,)
        for n in ("weight", "bias", "_mean", "_variance"):
            s[prefix + "bn." + n] = (cout,)
    for i in range(c["encoder_conv_layers"]):
        conv_bn(f"encoder.conv_batchnorms.{i}.", de, de, c["encoder_kernel_size"])
    h = de // 2
    for d in ("cell_fw", "cell_bw"):
        s[f"encoder.lstm.0.{d}.weight_ih"] = (4 * h, de)
        s[f"encoder.lstm.0.{d}.weight_hh"] = (4 * h, h)
        s[f"encoder.lstm.0.{d}.bias_ih"] = (4 * h,)
        s[f"encoder.lstm.0.{d}.bias_hh"] = (4 * h,)
    s["decoder.prenet.linear1.weight"] = (dm, c["d_prenet"])
    s["decoder.prenet.linear2.weight"] = (c["d_prenet"], c["d_prenet"])
    ha, hd = c["d_attention_rnn"], c["d_decoder_rnn"]
    for name, k_in, H in (("attention_rnn", c["d_prenet"] + dk, ha), ("decoder_rnn", ha + dk, hd)):
        s[f"decoder.{name}.weight_ih"] = (4 * H, k_in)
        s[f"decoder.{name}.weight_hh"] = (4 * H, H)
        s[f"decoder.{name}.bias_ih"] = (4 * H,)
        s[f"decoder.{name}.bias_hh"] = (4 * H,)
    a = "decoder.attention_layer."
    s[a + "query_layer.weight"] = (ha, c["d_attention"])
    s[a + "key_layer.weight"] = (dk, c["d_attention"])
    s[a + "value.weight"] = (c["d_attention"], 1)
    s[a + "location_conv.weight"] = (c["attention_filters"], 2, c["attention_kernel_size"])
    s[a + "location_layer.weight"] = (c["attention_filters"], c["d_attention"])
    s["decoder.linear_projection.weight"] = (hd + dk, dm)
    s["decoder.linear_projection.bias"] = (dm,)
    if c["use_stop_token"]:
        s["decoder.stop_layer.weight"] = (hd + dk, 1)
        s["decoder.stop_layer.bias"] = (1,)
    n = c["postnet_conv_layers"]
    for i in range(n):
        conv_bn(f"postnet.conv_batchnorms.{i}.", dm if i == 0 else c["d_postnet"], dm if i == n - 1 else c["d_postnet"],
                c["postnet_kernel_size"])
    return s


def synth_params(seed, cfg, stop_bias=None):
    """Random parameters of reference-like scale: uniform(+-1/sqrt(fan_in)), BatchNorm statistics near (0, 1)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, shape in param_shapes(cfg).items():
        if k.endswith("bn._mean"):
            v = torch.randn(shape, generator=g) * 0.1
        elif k.endswith("bn._variance"):
            v = torch.rand(shape, generator=g) + 0.5
        elif k.endswith("bn.weight"):
            v = torch.rand(shape, generator=g) + 0.5
        elif k.endswith("bn.bias"):
            v = (torch.rand(shape, generator=g) - 0.5) * 0.2
        elif k.startswith("embedding"):
            v = torch.randn(shape, generator=g) * 0.3
        else:
            if ".lstm." in k or "_rnn." in k:
                fan = shape[0] // 4                                        # Paddle's LSTM init: +-1/sqrt(hidden)
            elif len(shape) == 3:
                fan = shape[1] * shape[2]
            else:
                fan = shape[0]                                             # Linear [in, out]; 1-D biases use their size
            v = (torch.rand(shape, generator=g) * 2 - 1) / math.sqrt(fan)
        out[k] = v.float()
    if "embedding_tones.weight" in out:
        out["embedding_tones.weight"][0] = 0.0
    if stop_bias is not None and "decoder.stop_layer.bias" in out:
        out["decoder.stop_layer.bias"] = torch.full((1,), float(stop_bias))
    return out


def flat_lstm_keys(p):
    """The same parameters under the flat LSTM keys of later Paddle releases (weight_ih_l0, weight_ih_l0_reverse, ...)."""
    out = {}
    for k, v in p.items():
        if k.startswith("encoder.lstm.0."):
            d, part = k.split(".")[3], k.split(".")[4]
            out[f"encoder.lstm.{part}_l0" + ("_reverse" if d == "cell_bw" else "")] = v
        else:
            out[k] = v
    return out


def _drop(drop, site, x, p):
    """PhiloxDropout on x of any device (the mask is generated on the host)."""
    if p <= 0:
        return x
    keep = drop.keep_mask(site, x.numel(), p).reshape(x.shape).to(x.device)
    return x * keep * np.float32(1.0 / (1.0 - np.float32(p)))


def _conv_bn(p, prefix, x, dt):
    """Conv1dBatchNorm (NLC, 'same' padding, eval BatchNorm): x (B, T, C)."""
    w, b = p[prefix + "conv.weight"].to(dt), p[prefix + "conv.bias"].to(dt)
    y = torch.nn.functional.conv1d(x.transpose(1, 2), w, b, padding=(w.shape[2] - 1) // 2).transpose(1, 2)
    mean, var = p[prefix + "bn._mean"].to(dt), p[prefix + "bn._variance"].to(dt)
    return (y - mean) / torch.sqrt(var + 1e-5) * p[prefix + "bn.weight"].to(dt) + p[prefix + "bn.bias"].to(dt)


def _cell(p, prefix, x, h, c, dt):
    g = x @ p[prefix + "weight_ih"].to(dt).t() + p[prefix + "bias_ih"].to(dt) + h @ p[prefix + "weight_hh"].to(dt).t() + \
        p[prefix + "bias_hh"].to(dt)
    i, f, gg, o = g.chunk(4, dim=-1)
    c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
    return torch.sigmoid(o) * torch.tanh(c), c


def encoder(p, cfg, text, tones=None, text_lens=None, global_condition=None, dtype=torch.float64):
    """-> keys (B, T, d_encoder [+ d_global_condition]); rows past text_lens zero (they are masked out of every output)."""
    dt = dtype
    x = p["embedding.weight"].to(dt)[text.long()]
    if cfg["n_tones"]:
        tw = p["embedding_tones.weight"].to(dt).clone()
        tw[0] = 0.0
        x = x + tw[tones.long()]
    for i in range(cfg["encoder_conv_layers"]):
        x = torch.relu(_conv_bn(p, f"encoder.conv_batchnorms.{i}.", x, dt))
    B, T, _ = x.shape
    lens = [T] * B if text_lens is None else [int(v) for v in text_lens]
    H = cfg["d_encoder"] // 2
    out = torch.zeros(B, T, 2 * H, dtype=dt)
    for b in range(B):
        n = lens[b]
        for d, order in (("cell_fw", range(n)), ("cell_bw", range(n - 1, -1, -1))):
            h = torch.zeros(1, H, dtype=dt)
            c = torch.zeros(1, H, dtype=dt)
            for t in order:
                h, c = _cell(p, f"encoder.lstm.0.{d}.", x[b, t:t + 1], h, c, dt)
                out[b, t, (0 if d == "cell_fw" else H):(H if d == "cell_fw" else 2 * H)] = h[0]
    if global_condition is not None:
        gc = global_condition.to(dt).unsqueeze(1).expand(-1, T, -1)
        out = torch.cat([out, gc], -1)
        for b in range(B):
            out[b, lens[b]:] = 0.0
    return out


def decode(p, cfg, keys, *, mels=None, text_lens=None, max_decoder_steps=1000, seed=0, dtype=torch.float64):
    """Tacotron2Decoder.infer (mels None: frames fed back, the reference's stop rules) or .forward (teacher-forced on mels
    (B, T_mel, d_mels), energies masked with text_lens).  -> (mel (B, N, d_mels * r), align (B, N, T_enc), stop (B, N) or None)."""
    dt, dev = dtype, keys.device
    B, T_enc, dk = keys.shape
    r, dm = cfg["reduction_factor"], cfg["d_mels"] * cfg["reduction_factor"]
    ha, hd = cfg["d_attention_rnn"], cfg["d_decoder_rnn"]
    pdrop = cfg["p_prenet_dropout"]
    use_stop = cfg["use_stop_token"]
    a = "decoder.attention_layer."
    pkeys = keys @ p[a + "key_layer.weight"].to(dt)
    lw, ll = p[a + "location_conv.weight"].to(dt), p[a + "location_layer.weight"].to(dt)
    mask = None
    if mels is not None:
        steps = mels.shape[1] // r
        querys = mels.to(dt).reshape(B, steps, dm)
        if text_lens is not None:
            mask = (torch.arange(T_enc, device=dev)[None, :] < text_lens.to(dev).reshape(-1, 1).long()).to(dt)
    else:
        steps = max_decoder_steps
    z = lambda *shape: torch.zeros(*shape, dtype=dt, device=dev)
    h_a, c_a, h_d, c_d = z(B, ha), z(B, ha), z(B, hd), z(B, hd)
    w, wc, ctx, frame = z(B, T_enc), z(B, T_enc), z(B, dk), z(B, dm)
    mels_out, aligns, stops = [], [], []
    first_hit = None
    for i in range(steps):
        if mels is not None and i > 0:
            frame = querys[:, i - 1]
        drop = PhiloxDropout(seed, i)
        q = _drop(drop, PRENET_SITES[0], torch.relu(frame @ p["decoder.prenet.linear1.weight"].to(dt)), pdrop)
        q = _drop(drop, PRENET_SITES[1], torch.relu(q @ p["decoder.prenet.linear2.weight"].to(dt)), pdrop)
        h_a, c_a = _cell(p, "decoder.attention_rnn.", torch.cat([q, ctx], -1), h_a, c_a, dt)
        pq = h_a @ p[a + "query_layer.weight"].to(dt)
        loc = torch.nn.functional.conv1d(torch.stack([w, wc], 1), lw, padding=(lw.shape[2] - 1) // 2).transpose(1, 2) @ ll
        e = (torch.tanh(loc + pkeys + pq[:, None, :]) @ p[a + "value.weight"].to(dt))[..., 0]
        if mask is not None:
            e = e + (1.0 - mask) * -1e9
        w = torch.softmax(e, dim=1)
        ctx = torch.einsum("bt,btc->bc", w, keys)
        wc = wc + w
        h_d, c_d = _cell(p, "decoder.decoder_rnn.", torch.cat([h_a, ctx], -1), h_d, c_d, dt)
        z = torch.cat([h_d, ctx], -1)
        frame = z @ p["decoder.linear_projection.weight"].to(dt) + p["decoder.linear_projection.bias"].to(dt)
        mels_out.append(frame)
        aligns.append(w)
        if use_stop:
            stops.append((z @ p["decoder.stop_layer.weight"].to(dt) + p["decoder.stop_layer.bias"].to(dt))[:, 0])
        if mels is None:
            if use_stop:
                if torch.sigmoid(stops[-1][0].float()) > 0.5:
                    break
            elif int(torch.argmax(w[0])) == T_enc - 1:
                if first_hit is None:
                    first_hit = i
                elif i > first_hit + 20:
                    break
    return torch.stack(mels_out, 1), torch.stack(aligns, 1), (torch.stack(stops, 1) if use_stop else None)


def postnet(p, cfg, mel, dtype=torch.float64):
    """mel + DecoderPostNet(mel) (eval)."""
    x = mel.to(dtype)
    n = cfg["postnet_conv_layers"]
    for i in range(n):
        x = _conv_bn(p, f"postnet.conv_batchnorms.{i}.", x, dtype)
        if i < n - 1:
            x = torch.tanh(x)
    return mel.to(dtype) + x


def forward(p, cfg, text, text_lens, mels, output_lens=None, tones=None, global_condition=None, seed=0, dtype=torch.float64):
    keys = encoder(p, cfg, text, tones, text_lens, global_condition, dtype)
    mel, align, stop = decode(p, cfg, keys, mels=mels, text_lens=text_lens, seed=seed, dtype=dtype)
    post = postnet(p, cfg, mel, dtype)
    if output_lens is not None:
        m = (torch.arange(mel.shape[1])[None, :] < output_lens.reshape(-1, 1).long()).to(dtype)[..., None]
        mel, post = mel * m, post * m
    out = {"mel_output": mel, "mel_outputs_postnet": post, "alignments": align}
    if stop is not None:
        out["stop_logits"] = stop
    return out


def infer(p, cfg, text, max_decoder_steps=1000, tones=None, global_condition=None, seed=0, dtype=torch.float64):
    keys = encoder(p, cfg, text, tones, None, global_condition, dtype)
    mel, align, stop = decode(p, cfg, keys, max_decoder_steps=max_decoder_steps, seed=seed, dtype=dtype)
    out = {"mel_output": mel, "mel_outputs_postnet": postnet(p, cfg, mel, dtype), "alignments": align}
    if stop is not None:
        out["stop_logits"] = stop
    return out


def loss(mel, post, target, align=None, slens=None, plens=None, stop_logits=None, use_stop_token_loss=True,
         use_guided_attention_loss=False, sigma=0.2):
    """Tacotron2Loss.forward in the dtype of the inputs -> dict."""
    mel_loss = ((mel - target) ** 2).mean()
    post_loss = ((post - target) ** 2).mean()
    total = mel_loss + post_loss
    out = {"mel_loss": mel_loss, "post_mel_loss": post_loss}
    if use_guided_attention_loss:
        _, N, T = align.shape
        dec = slens.to(align.dtype).reshape(-1, 1)
        enc = plens.to(align.dtype).reshape(-1, 1)
        W = 1 - torch.exp(-((torch.arange(N, dtype=align.dtype) / dec)[:, :, None] - (torch.arange(T, dtype=align.dtype) / enc)[:, None, :])
                          ** 2 / (2 * sigma ** 2))
        m = (torch.arange(N)[None, :] < slens.reshape(-1, 1)).to(align.dtype)[:, :, None] * \
            (torch.arange(T)[None, :] < plens.reshape(-1, 1)).to(align.dtype)[:, None, :]
        gal = ((W * m * align).sum((1, 2)) / (slens * plens).to(align.dtype)).mean()
        total = total + gal
        out["guided_attn_loss"] = gal
    if use_stop_token_loss:
        T_dec = target.shape[1]
        labels = torch.nn.functional.one_hot((slens - 1).long(), T_dec).to(stop_logits.dtype)
        st = torch.nn.functional.binary_cross_entropy_with_logits(stop_logits, labels)
        total = total + st
        out["stop_loss"] = st
    out["loss"] = total
    return out


def synth_text(seed, batch, length, vocab, n_tones=None):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(0, vocab, (batch, length), generator=g)
    tones = torch.randint(1, n_tones, (batch, length), generator=g) if n_tones else None
    return text, tones

