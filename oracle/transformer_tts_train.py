"""TransformerTTS training step restated in torch (reference: TransformerTTSUpdater.update_core,
parakeet/models/transformer_tts/transformer_tts_updater.py:73-170): the train-mode forward with Dropout at the step's sites,
TransformerTTSLoss (transformer_tts.py:770-872), GuidedMultiHeadAttentionLoss on the source attention (:874-1075), torch autograd for
loss.backward(); paddle.optimizer.Adam is oracle.fastspeech2.adam_step.  The model's eval-mode pieces, configs and seeded weights are
oracle.transformer_tts's.
"""
import math

import torch

from . import fastspeech2 as ofs
from .transformer_tts import LJSPEECH, P_PRENET, SMALL, eos_and_labels, golden_batch, synth_params  # noqa: F401

# the training golden (scripts/make_golden_ref.py transformer_tts_train): SMALL at r = 1 with every transformer and postnet dropout
# rate 0 (the prenet's always-on masks are the step's, seed TRAIN_SEED, step 1) and the recipe's guided-loss lambda
TRAIN_SMALL = dict(SMALL, reduction_factor=1, transformer_enc_dropout_rate=0.0, transformer_enc_positional_dropout_rate=0.0,
                   transformer_enc_attn_dropout_rate=0.0, transformer_dec_dropout_rate=0.0, transformer_dec_positional_dropout_rate=0.0,
                   transformer_dec_attn_dropout_rate=0.0, transformer_enc_dec_attn_dropout_rate=0.0, postnet_dropout_rate=0.0)
TRAIN_SEED, TRAIN_LAMBDA = 5, 10.0


def dropout_site(stack, layer, kind):
    """Site numbering shared with parakeet_b200/training/transformer_tts_step.py: stack * 1000 + layer * 10 + kind.  stack: 0 encoder,
    1 decoder, 2 decoder prenet, 5 postnet; kind: 0 positional encoding, 1 self-attention probabilities, 2 self-attention
    sub-layer output, 3 feed-forward hidden, 4 feed-forward sub-layer output, 5 source-attention probabilities, 6 source-attention
    sub-layer output (decoder) or postnet layer (stack 5), 7 prenet layer.  The encoder's sites are oracle.fastspeech2's."""
    return ofs.dropout_site(stack, layer, kind)


def train_prenet_masks(seed, step, batch, rows, units, n_layers, p=P_PRENET):
    """The training step's prenet keep masks (n_layers, batch, rows, units): pk_dropout's Philox at site dropout_site(2, i, 7) and
    step `step` (1 + completed steps), element index (b * rows + t) * units + j."""
    d = ofs.PhiloxDropout(seed, step)
    return torch.stack([d.keep_mask(dropout_site(2, i, 7), batch * rows * units, p).reshape(batch, rows, units) for i in range(n_layers)])


def _mha_train(p, pre, q_in, kv_in, n_head, mask, dropout, site, rate):
    """MultiHeadedAttention in train mode -> (output, the pre-dropout weights (B, H, Tq, Tk)); dropout on the weights in the CUDA
    layout (B * H, Tq, ceil64(Tk))."""
    B, Tq, A = q_in.shape
    dk = A // n_head
    q = ofs.linear(p, pre + "linear_q", q_in).reshape(B, Tq, n_head, dk).transpose(1, 2)
    k = ofs.linear(p, pre + "linear_k", kv_in).reshape(B, -1, n_head, dk).transpose(1, 2)
    v = ofs.linear(p, pre + "linear_v", kv_in).reshape(B, -1, n_head, dk).transpose(1, 2)
    Tk = k.shape[2]
    m = ~mask.unsqueeze(1)
    scores = (torch.matmul(q, k.transpose(-2, -1)) / math.sqrt(dk)).masked_fill(m, torch.finfo(torch.float32).min)
    att = torch.softmax(scores, dim=-1).masked_fill(m, 0.0)
    ad = att
    if dropout is not None and rate > 0:
        Tp = (Tk + 63) // 64 * 64
        padded = torch.nn.functional.pad(att, (0, Tp - Tk)).reshape(B * n_head, Tq, Tp)
        ad = dropout(site, padded, rate).reshape(B, n_head, Tq, Tp)[..., :Tk]
    return ofs.linear(p, pre + "linear_out", torch.matmul(ad, v).transpose(1, 2).reshape(B, Tq, A)), att


def train_forward(p, cfg, text, text_lens, speech, speech_lens, prenet_keep, dropout=None, rates=None):
    """TransformerTTS.forward in train mode (r = 1) -> dict as `forward`, plus new_stats (the postnet's running statistics).
    prenet_keep: keep masks (n_layers, B, L, units) of the always-on prenet dropout; dropout: None (every other rate 0) or a
    oracle.fastspeech2.PhiloxDropout with `rates` (the reference's keywords)."""
    R = {k: 0.0 for k in ("transformer_enc_dropout_rate", "transformer_enc_positional_dropout_rate", "transformer_enc_attn_dropout_rate",
                          "transformer_dec_dropout_rate", "transformer_dec_positional_dropout_rate", "transformer_dec_attn_dropout_rate",
                          "transformer_enc_dec_attn_dropout_rate", "postnet_dropout_rate")}
    R.update(rates or {})
    drop = (lambda site, x, rate: x if dropout is None or rate <= 0 else dropout(site, x, rate))
    odim, H = cfg["odim"], cfg["aheads"]
    xs, ilens, labels, olens = eos_and_labels(text, text_lens, speech_lens, cfg["idim"] - 1, 1)
    B, Tk = xs.shape
    hs = ofs.encoder(p, "encoder.", xs, ofs.make_non_pad_mask(ilens, Tk).unsqueeze(1), cfg["elayers"], H, dropout=dropout, stack=0,
                     rates=(R["transformer_enc_dropout_rate"], R["transformer_enc_positional_dropout_rate"], R["transformer_enc_attn_dropout_rate"]))
    ys = speech
    Lr = ys.shape[1]
    h = torch.cat([torch.zeros_like(ys[:, :1]), ys[:, :-1]], 1)
    for i in range(cfg["dprenet_layers"]):
        h = torch.relu(ofs.linear(p, f"decoder.embed.0.0.prenet.{i}.0", h)) * prenet_keep[i].to(h) * (1.0 / (1.0 - P_PRENET))
    x = ofs.linear(p, "decoder.embed.0.1", h)
    x = x + p["decoder.embed.1.alpha"] * ofs.positional_encoding(Lr, x.shape[2]).to(x)
    x = drop(dropout_site(1, 0, 0), x, R["transformer_dec_positional_dropout_rate"])
    y_mask = ofs.make_non_pad_mask(speech_lens, Lr).unsqueeze(1) & torch.tril(torch.ones(Lr, Lr, dtype=torch.bool)).unsqueeze(0)
    m_mask = ofs.make_non_pad_mask(ilens, Tk).unsqueeze(1)
    r_layer = R["transformer_dec_dropout_rate"]
    atts = []
    for l in range(cfg["dlayers"]):
        q = f"decoder.decoders.{l}."
        tn = ofs.layer_norm(p, q + "norm1", x)
        a, _ = _mha_train(p, q + "self_attn.", tn, tn, H, y_mask, dropout, dropout_site(1, l, 1), R["transformer_dec_attn_dropout_rate"])
        x = x + drop(dropout_site(1, l, 2), a, r_layer)
        a, w = _mha_train(p, q + "src_attn.", ofs.layer_norm(p, q + "norm2", x), hs, H, m_mask, dropout, dropout_site(1, l, 5),
                          R["transformer_enc_dec_attn_dropout_rate"])
        x = x + drop(dropout_site(1, l, 6), a, r_layer)
        atts.append(w)
        u = drop(dropout_site(1, l, 3), torch.relu(ofs.linear(p, q + "feed_forward.w_1", ofs.layer_norm(p, q + "norm3", x))), r_layer)
        x = x + drop(dropout_site(1, l, 4), ofs.linear(p, q + "feed_forward.w_2", u), r_layer)
    zs = ofs.layer_norm(p, "decoder.after_norm", x)
    before = ofs.linear(p, "feat_out", zs).reshape(B, -1, odim)
    logits = ofs.linear(p, "prob_out", zs).reshape(B, -1)
    new_stats = {}
    post = ofs.postnet(p, before.transpose(1, 2), cfg["postnet_layers"], train_bn=True, new_stats=new_stats, dropout=dropout,
                       rate=R["postnet_dropout_rate"])
    after = before + post.transpose(1, 2)
    return dict(after_outs=after, before_outs=before, logits=logits, ys=ys, labels=labels, olens=olens, ilens=ilens,
                att_ws=torch.stack(atts, 1), new_stats=new_stats)


def tts_loss(after, before, logits, ys, labels, olens, pos_weight=5.0):
    """TransformerTTSLoss (use_masking=True) -> (l1, l2, bce) over the frames t < olens[b]."""
    mask = ofs.make_non_pad_mask(olens, ys.shape[1])
    m3 = mask.unsqueeze(-1).expand_as(ys)
    a, b, y = after[m3], before[m3], ys[m3]
    l1 = (a - y).abs().mean() + (b - y).abs().mean()
    l2 = ((a - y) ** 2).mean() + ((b - y) ** 2).mean()
    bce = torch.nn.functional.binary_cross_entropy_with_logits(logits[mask], labels[mask].to(logits), pos_weight=torch.tensor(pos_weight).to(logits))
    return l1, l2, bce


def guided_mask(ilen, olen, sigma=0.4):
    """GuidedAttentionLoss._make_guided_attention_mask: (olen, ilen) = 1 - exp(-(j / ilen - i / olen)^2 / (2 sigma^2)), in fp32."""
    gx, gy = torch.meshgrid(torch.arange(olen, dtype=torch.float32), torch.arange(ilen, dtype=torch.float32), indexing="ij")
    return 1.0 - torch.exp(-((gy / ilen - gx / olen) ** 2) / (2 * (sigma ** 2)))


def guided_attn_loss(att_ws, ilens, olens, sigma=0.4, alpha=1.0):
    """GuidedMultiHeadAttentionLoss: att_ws (B, heads x layers, T_out, T_in) -> alpha * mean of G * att over the non-pad elements."""
    B, _, To, Ti = att_ws.shape
    G = torch.zeros(B, To, Ti, dtype=att_ws.dtype)
    for b in range(B):
        i, o = int(ilens[b]), int(olens[b])
        G[b, :o, :i] = guided_mask(i, o, sigma).to(att_ws.dtype)
    masks = ofs.make_non_pad_mask(olens, To).unsqueeze(-1) & ofs.make_non_pad_mask(ilens, Ti).unsqueeze(-2)
    losses = G.unsqueeze(1) * att_ws
    return alpha * losses.masked_select(masks.unsqueeze(1).expand_as(losses)).mean()


def train_step_grads(p, cfg, batch, prenet_keep, dropout=None, rates=None, loss_type="L1", pos_weight=5.0, sigma=0.4, lam=1.0,
                     guided=True, dtype=torch.float64):
    """update_core up to loss.backward() -> (losses dict of floats, grads dict keyed like p (trainable tensors), new BN stats)."""
    q = {k: (v.to(dtype).clone().requires_grad_(True) if not k.endswith(ofs.BUFFER_SUFFIXES) else v.to(dtype).clone()) for k, v in p.items()}
    out = train_forward(q, cfg, batch["text"], batch["text_lengths"], batch["speech"].to(dtype), batch["speech_lengths"], prenet_keep,
                        dropout, rates)
    l1, l2, bce = tts_loss(out["after_outs"], out["before_outs"], out["logits"], out["ys"], out["labels"], out["olens"], pos_weight)
    loss = {"L1": l1, "L2": l2, "L1+L2": l1 + l2}[loss_type] + bce
    res = dict(l1_loss=l1, l2_loss=l2, bce_loss=bce)
    if guided:
        nh, nl = cfg["num_heads_applied_guided_attn"], cfg["num_layers_applied_guided_attn"]
        att = torch.cat([out["att_ws"][:, l, :nh] for l in reversed(range(cfg["dlayers"]))][:nl], 1)
        g = guided_attn_loss(att, out["ilens"], out["olens"], sigma, lam)
        res["enc_dec_attn_loss"] = g
        loss = loss + g
    res["loss"] = loss
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in q.items() if not k.endswith(ofs.BUFFER_SUFFIXES)}
    return {k: float(v.detach()) for k, v in res.items()}, grads, out["new_stats"]
