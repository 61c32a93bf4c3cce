"""TransformerTTS restated in torch (reference: parakeet/models/transformer_tts/transformer_tts.py `TransformerTTS.inference`,
modules/fastspeech2_transformer/decoder.py `Decoder.forward_one_step`, decoder_layer.py `DecoderLayer.forward` with a cache,
modules/tacotron2/decoder.py `Prenet` / `Postnet`).

`inference` is `encode`, then `decode`, the reference's own step loop on the encoder output: every step re-embeds every earlier frame through the prenet, and each decoder layer
computes only the new query row over [its cached outputs | the new row], exactly as `forward_one_step` does; no K / V cache of its own.

The prenet's `F.dropout` is always on with Paddle's default p = 0.5 (it ignores `dprenet_dropout_rate`).  Its masks cannot be
reproduced from Paddle's generator; here (and in pk_tts_decode) they are Philox masks keyed by frame position: prenet layer i is
site i, the frame's row in the decoder input is the Philox step and the element is b * units + j (oracle.fastspeech2.PhiloxDropout).
"""
import math

import torch

from . import fastspeech2 as ofs

# examples/transformer_tts/ljspeech/conf/default.yaml (model:) with idim / odim of the recipe
LJSPEECH = dict(idim=78, odim=80, embed_dim=0, eprenet_conv_layers=0, eprenet_conv_filts=0, eprenet_conv_chans=0, dprenet_layers=2,
                dprenet_units=256, adim=512, aheads=8, elayers=6, eunits=1024, dlayers=6, dunits=1024, positionwise_layer_type="conv1d",
                positionwise_conv_kernel_size=1, postnet_layers=5, postnet_filts=5, postnet_chans=256, use_scaled_pos_enc=True,
                encoder_normalize_before=True, decoder_normalize_before=True, reduction_factor=1, init_type="xavier_uniform",
                init_enc_alpha=1.0, init_dec_alpha=1.0, eprenet_dropout_rate=0.0, dprenet_dropout_rate=0.5, postnet_dropout_rate=0.5,
                transformer_enc_dropout_rate=0.1, transformer_enc_positional_dropout_rate=0.1, transformer_enc_attn_dropout_rate=0.1,
                transformer_dec_dropout_rate=0.1, transformer_dec_positional_dropout_rate=0.1, transformer_dec_attn_dropout_rate=0.1,
                transformer_enc_dec_attn_dropout_rate=0.1, num_heads_applied_guided_attn=2, num_layers_applied_guided_attn=2)
# a small config of the same structure: 2 + 2 layers, adim 128 in two 64-wide heads, r = 2, a 3-tap encoder FFN
SMALL = dict(LJSPEECH, idim=20, odim=8, dprenet_units=32, adim=128, aheads=2, elayers=2, eunits=64, dlayers=2, dunits=96,
             postnet_chans=16, reduction_factor=2, positionwise_conv_kernel_size=3)
GOLDEN_CONFIGS = {"small": (SMALL, 11), "ljspeech": (LJSPEECH, 12)}
P_PRENET = 0.5          # F.dropout's default in DecoderPrenet.forward, whatever dprenet_dropout_rate says


def param_shapes(cfg):
    """The reference's state-dict keys and shapes (Paddle Linear [in, out], Conv1D [out, in, k]) for the supported configs."""
    A, U, k = cfg["adim"], cfg["eunits"], cfg["positionwise_conv_kernel_size"]
    s = {"encoder.embed.0.weight": (cfg["idim"], A), "encoder.embed.1.alpha": (1,)}

    def attn(pre):
        for n in ("linear_q", "linear_k", "linear_v", "linear_out"):
            s[f"{pre}{n}.weight"], s[f"{pre}{n}.bias"] = (A, A), (A,)

    for i in range(cfg["elayers"]):
        q = f"encoder.encoders.{i}."
        attn(q + "self_attn.")
        s[q + "feed_forward.w_1.weight"], s[q + "feed_forward.w_1.bias"] = (U, A, k), (U,)
        s[q + "feed_forward.w_2.weight"], s[q + "feed_forward.w_2.bias"] = (A, U, k), (A,)
        for n in ("norm1", "norm2"):
            s[f"{q}{n}.weight"], s[f"{q}{n}.bias"] = (A,), (A,)
    s["encoder.after_norm.weight"], s["encoder.after_norm.bias"] = (A,), (A,)
    Up = cfg["dprenet_units"]
    for i in range(cfg["dprenet_layers"]):
        s[f"decoder.embed.0.0.prenet.{i}.0.weight"] = (cfg["odim"] if i == 0 else Up, Up)
        s[f"decoder.embed.0.0.prenet.{i}.0.bias"] = (Up,)
    s["decoder.embed.0.1.weight"], s["decoder.embed.0.1.bias"] = (Up, A), (A,)
    s["decoder.embed.1.alpha"] = (1,)
    D = cfg["dunits"]
    for i in range(cfg["dlayers"]):
        q = f"decoder.decoders.{i}."
        attn(q + "self_attn.")
        attn(q + "src_attn.")
        s[q + "feed_forward.w_1.weight"], s[q + "feed_forward.w_1.bias"] = (A, D), (D,)
        s[q + "feed_forward.w_2.weight"], s[q + "feed_forward.w_2.bias"] = (D, A), (A,)
        for n in ("norm1", "norm2", "norm3"):
            s[f"{q}{n}.weight"], s[f"{q}{n}.bias"] = (A,), (A,)
    s["decoder.after_norm.weight"], s["decoder.after_norm.bias"] = (A,), (A,)
    r, odim = cfg["reduction_factor"], cfg["odim"]
    s["feat_out.weight"], s["feat_out.bias"] = (A, odim * r), (odim * r,)
    s["prob_out.weight"], s["prob_out.bias"] = (A, r), (r,)
    n, C = cfg["postnet_layers"], cfg["postnet_chans"]
    for i in range(n):
        ci, co = (odim if i == 0 else C), (odim if i == n - 1 else C)
        s[f"postnet.postnet.{i}.0.weight"] = (co, ci, cfg["postnet_filts"])
        for b in ("weight", "bias", "_mean", "_variance"):
            s[f"postnet.postnet.{i}.1.{b}"] = (co,)
    return s


def synth_params(seed, cfg, prob_bias=-4.0):
    """Seeded weights with the reference's keys: uniform(+-1/sqrt(fan_in)) matrices, small biases, LayerNorm / BatchNorm near
    identity, alphas 1; prob_out's bias at `prob_bias` (the stop probability starts low)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, shape in param_shapes(cfg).items():
        if k.endswith("alpha"):
            v = torch.ones(shape)
        elif k.endswith("_variance"):
            v = 1.0 + 0.2 * torch.rand(shape, generator=g)
        elif k.endswith("_mean") or k.endswith(".bias"):
            v = 0.05 * torch.randn(shape, generator=g)
        elif ("norm" in k or ".1.weight" in k and k.startswith("postnet")) and len(shape) == 1:
            v = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            fan = shape[0] if len(shape) == 2 else shape[1] * shape[2]
            v = (torch.rand(shape, generator=g) * 2 - 1) / math.sqrt(fan)
        out[k] = v.float()
    out["encoder.embed.0.weight"][0] = 0.0                      # padding_idx row
    out["prob_out.bias"] = torch.full((cfg["reduction_factor"],), float(prob_bias))
    return out


def prenet_masks(seed, rows, units, n_layers, batch=1, p=P_PRENET):
    """Keep masks (n_layers, batch, rows, units) float: site = layer, Philox step = row, element = b * units + j."""
    out = torch.empty(n_layers, batch, rows, units)
    for t in range(rows):
        d = ofs.PhiloxDropout(seed, t)
        for i in range(n_layers):
            out[i, :, t] = d.keep_mask(i, batch * units, p).reshape(batch, units)
    return out


def _mha(p, pre, q_in, kv_in, n_head, mask=None):
    """MultiHeadedAttention(query, key, value, mask) -> (output (B, Tq, A), weights (B, H, Tq, Tk)); mask bool (B, 1 or Tq, Tk), True
    where a key is attended (forward_attention: masked_fill(min) -> softmax -> masked_fill(0))."""
    B, Tq, A = q_in.shape
    dk = A // n_head
    q = ofs.linear(p, pre + "linear_q", q_in).reshape(B, Tq, n_head, dk).transpose(1, 2)
    k = ofs.linear(p, pre + "linear_k", kv_in).reshape(B, -1, n_head, dk).transpose(1, 2)
    v = ofs.linear(p, pre + "linear_v", kv_in).reshape(B, -1, n_head, dk).transpose(1, 2)
    scores = torch.matmul(q, k.transpose(-2, -1)) / math.sqrt(dk)
    if mask is None:
        att = torch.softmax(scores, dim=-1)
    else:
        m = ~mask.unsqueeze(1)
        att = torch.softmax(scores.masked_fill(m, torch.finfo(torch.float32).min), dim=-1).masked_fill(m, 0.0)
    return ofs.linear(p, pre + "linear_out", torch.matmul(att, v).transpose(1, 2).reshape(B, Tq, A)), att


def encode(p, cfg, text):
    """Encoder(xs, None) on one utterance (1, T) int64 that already ends with eos -> hs (1, T, adim)."""
    return ofs.encoder(p, "encoder.", text, None, cfg["elayers"], cfg["aheads"])


def embed_frames(p, cfg, ys, keep):
    """decoder.embed: DecoderPrenet (Linear -> ReLU -> dropout with the given keep masks (layers, 1, rows, units)), Linear, + alpha pe."""
    h = ys
    for i in range(cfg["dprenet_layers"]):
        h = torch.relu(ofs.linear(p, f"decoder.embed.0.0.prenet.{i}.0", h))
        h = h * keep[i, :, :h.shape[1]].to(h) * (1.0 / (1.0 - P_PRENET))
    x = ofs.linear(p, "decoder.embed.0.1", h)
    return x + p["decoder.embed.1.alpha"] * ofs.positional_encoding(x.shape[1], x.shape[2]).to(x)


def inference(p, cfg, text, threshold=0.5, minlenratio=0.0, maxlenratio=10.0, seed=0, dtype=torch.float64):
    """TransformerTTS.inference (no teacher forcing) on text (T,) int64 without eos -> (outs (L r, odim), probs (L r,),
    att_ws (dlayers, aheads, L, T + 1), the per-step decoder outputs before the postnet (L r, odim))."""
    p = {k: v.to(dtype) for k, v in p.items()}
    r = cfg["reduction_factor"]
    x = torch.cat([text.reshape(-1).long(), torch.tensor([cfg["idim"] - 1])]).unsqueeze(0)
    hs = encode(p, cfg, x)
    maxlen = int(hs.shape[1] * maxlenratio / r)
    minlen = int(hs.shape[1] * minlenratio / r)
    before, probs, att_ws = decode(p, cfg, hs, minlen, maxlen, threshold, seed, dtype)
    after = before + ofs.postnet(p, before.t().unsqueeze(0), cfg["postnet_layers"])[0].t()
    return after, probs, att_ws, before


def decode(p, cfg, hs, minlen, maxlen, threshold, seed, dtype=torch.float64):
    """inference's decoder loop on the encoder output hs (1, T, adim), on hs's device -> (the decoder outputs before the postnet
    (L r, odim), probs (L r,), att_ws (dlayers, aheads, L, T)); it stops after step idx once (any prob >= threshold or
    idx >= maxlen) and idx >= minlen."""
    p = {k: v.to(hs.device, dtype) for k, v in p.items()}
    hs = hs.to(dtype)
    r, odim, H = cfg["reduction_factor"], cfg["odim"], cfg["aheads"]
    cap = max(maxlen, minlen, 1)
    keep = prenet_masks(seed, cap, cfg["dprenet_units"], cfg["dprenet_layers"]) if P_PRENET > 0 else None
    ys = torch.zeros(1, 1, odim, dtype=dtype, device=hs.device)
    cache = [None] * cfg["dlayers"]
    outs, probs, att_ws = [], [], []
    idx = 0
    while True:
        idx += 1
        xd = embed_frames(p, cfg, ys, keep)
        new_cache, atts = [], []
        for l in range(cfg["dlayers"]):
            q = f"decoder.decoders.{l}."
            tn = ofs.layer_norm(p, q + "norm1", xd)
            a, _ = _mha(p, q + "self_attn.", tn[:, -1:], tn, H)
            y = xd[:, -1:] + a
            a, w = _mha(p, q + "src_attn.", ofs.layer_norm(p, q + "norm2", y), hs, H)
            y = y + a
            f = ofs.linear(p, q + "feed_forward.w_2", torch.relu(ofs.linear(p, q + "feed_forward.w_1", ofs.layer_norm(p, q + "norm3", y))))
            y = y + f
            xd = y if cache[l] is None else torch.cat([cache[l], y], 1)
            new_cache.append(xd)
            atts.append(w[0, :, -1])                                  # (H, T)
        cache = new_cache
        z = ofs.layer_norm(p, "decoder.after_norm", xd[:, -1])
        outs.append(ofs.linear(p, "feat_out", z).reshape(r, odim))
        probs.append(torch.sigmoid(ofs.linear(p, "prob_out", z))[0])
        att_ws.append(torch.stack(atts))                              # (layers, H, T)
        ys = torch.cat([ys, outs[-1][-1].reshape(1, 1, odim)], 1)
        if bool((probs[-1] >= threshold).any()) or idx >= maxlen:
            if idx < minlen:
                continue
            break
    return torch.cat(outs, 0), torch.cat(probs, 0), torch.stack(att_ws, 2)


def golden_text(cfg, seed, n):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(1, cfg["idim"] - 1, (n,), generator=g)


def eos_and_labels(text, text_lens, speech_lens, eos, r):
    """The reference forward's host-side construction: (xs (B, T + 1) with eos at column text_lens[b], ilens, labels, olens) with
    labels = pad(make_pad_mask(olens - 1), 1 column of ones), cut to max(olens - olens % r) with its last column 1 when r > 1."""
    xs = torch.nn.functional.pad(text.long(), (0, 1))
    for b, n in enumerate(text_lens.tolist()):
        xs[b, n] = eos
    olens = speech_lens.long()
    labels = torch.nn.functional.pad(ofs.make_pad_mask(olens - 1).float(), (0, 1), value=1.0)
    if r > 1:
        olens = olens - olens % r
        labels = labels[:, :int(olens.max())].clone()
        labels[:, -1] = 1.0
    return xs, text_lens.long() + 1, labels, olens


def forward(p, cfg, text, text_lens, speech, speech_lens, seed=0, dtype=torch.float64):
    """TransformerTTS.forward (eval; prenet dropout with the position-keyed masks) -> dict of after_outs, before_outs, logits, ys,
    labels, olens, ilens and the source attention weights att_ws (B, dlayers, aheads, L // r, T + 1).  Padded query rows are live."""
    p = {k: v.to(dtype) for k, v in p.items()}
    r, odim, H = cfg["reduction_factor"], cfg["odim"], cfg["aheads"]
    xs, ilens, labels, olens = eos_and_labels(text, text_lens, speech_lens, cfg["idim"] - 1, r)
    B, Tk = xs.shape
    hs = ofs.encoder(p, "encoder.", xs, ofs.make_non_pad_mask(ilens, Tk).unsqueeze(1), cfg["elayers"], H)
    ys = speech.to(dtype)
    ys_in = ys[:, r - 1::r]
    ys_in = torch.cat([torch.zeros_like(ys_in[:, :1]), ys_in[:, :-1]], 1)
    Lr = ys_in.shape[1]
    olens_in = speech_lens.long() // r
    keep = prenet_masks(seed, Lr, cfg["dprenet_units"], cfg["dprenet_layers"], batch=B)
    x = embed_frames(p, cfg, ys_in, keep)
    y_mask = ofs.make_non_pad_mask(olens_in, Lr).unsqueeze(1) & torch.tril(torch.ones(Lr, Lr, dtype=torch.bool)).unsqueeze(0)
    m_mask = ofs.make_non_pad_mask(ilens, Tk).unsqueeze(1)
    atts = []
    for l in range(cfg["dlayers"]):
        q = f"decoder.decoders.{l}."
        tn = ofs.layer_norm(p, q + "norm1", x)
        x = x + _mha(p, q + "self_attn.", tn, tn, H, y_mask)[0]
        a, w = _mha(p, q + "src_attn.", ofs.layer_norm(p, q + "norm2", x), hs, H, m_mask)
        x = x + a
        atts.append(w)
        x = x + ofs.linear(p, q + "feed_forward.w_2", torch.relu(ofs.linear(p, q + "feed_forward.w_1", ofs.layer_norm(p, q + "norm3", x))))
    zs = ofs.layer_norm(p, "decoder.after_norm", x)
    before = ofs.linear(p, "feat_out", zs).reshape(B, -1, odim)
    logits = ofs.linear(p, "prob_out", zs).reshape(B, -1)
    after = before + ofs.postnet(p, before.transpose(1, 2), cfg["postnet_layers"]).transpose(1, 2)
    if r > 1:
        ys = ys[:, :int(olens.max())]
    return dict(after_outs=after, before_outs=before, logits=logits, ys=ys, labels=labels, olens=olens, ilens=ilens,
                att_ws=torch.stack(atts, 1))


def golden_batch(cfg, seed, lens=(9, 4, 1), frames=(14, 9, 6)):
    """A ragged batch: text (B, max lens) ids in [1, idim - 1) zero padded, speech (B, max frames, odim) with garbage (not zeros) in
    the padded frames, as a padded data loader may leave it."""
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    text = torch.zeros(B, max(lens), dtype=torch.int64)
    for b, n in enumerate(lens):
        text[b, :n] = torch.randint(1, cfg["idim"] - 1, (n,), generator=g)
    speech = torch.randn(B, max(frames), cfg["odim"], generator=g) * 0.5
    return text, torch.tensor(lens), speech, torch.tensor(frames)
