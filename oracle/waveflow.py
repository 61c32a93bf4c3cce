"""Oracle: ConditionalWaveFlow inference (torch-CPU fp32 restatement).  TEST INFRASTRUCTURE ONLY.

Follows /root/reference/parakeet/models/waveflow.py:
  fold :32-51; UpsampleNet.forward :103-132 (Conv2DTranspose(1,1,(3,2f),stride(1,f),padding(1,f//2)), trim, leaky_relu 0.4)
  ResidualBlock.add_input / _update_buffer :228-294 (3-row causal buffer, Conv2D dilation (dh, 2^i), width "same" padding)
  ResidualNet.add_input :368-392; Flow._predict_row_parameters / _inverse_row / inverse :496-556
  WaveFlow._create_perm :602-615, _trim :617-625, inverse :674-711; ConditionalWaveFlow.infer :784-805 (z supplied by caller)
and parakeet/modules/geometry.py:18-50 (shuffle_dim = gather along H).
Paddle layouts: Conv2D weight [out, in, kh, kw]; Conv2DTranspose weight [in, out, kh, kw]; weight_norm g is 1-D [out]
(for Conv2DTranspose paddle normalises over dim 0 as well, i.e. per *input* channel - 1 channel here, so g is a scalar [1]).
"""
import math

import torch
import torch.nn.functional as F

DILATIONS_H = {8: [1] * 8, 16: [1] * 8, 32: [1, 2, 4, 1, 2, 4, 1, 2], 64: [1, 2, 4, 8, 16, 1, 2, 4], 128: [1, 2, 4, 8, 16, 32, 64, 1]}


def fold_weight_norm(params):
    out = {}
    for k, v in params.items():
        if k.endswith("weight_g"):
            continue
        if k.endswith("weight_v"):
            g = params[k[:-1] + "g"]
            norm = v.reshape(v.shape[0], -1).norm(dim=1)
            out[k[:-2]] = v * (g / norm).reshape([-1] + [1] * (v.dim() - 1))
        else:
            out[k] = v
    return out


def encoder(p, mel, n_up, trim_conv_artifact=True):
    """UpsampleNet.forward (:103-132): mel (B, C, T') -> (B, C, T)."""
    x = mel.unsqueeze(1)
    for i in range(n_up):
        w, b = p[f"encoder.{i}.weight"], p[f"encoder.{i}.bias"]
        f = w.shape[-1] // 2
        x = F.conv_transpose2d(x, w, b, stride=(1, f), padding=(1, f // 2))
        if trim_conv_artifact:
            x = x[:, :, :, :-(w.shape[-1] - f)]
        x = F.leaky_relu(x, 0.4)
    return x.squeeze(1)


def create_perm(n_group, n_flows):
    idx = list(range(n_group))
    half = n_group // 2
    return [idx[::-1] if i < n_flows // 2 else list(reversed(idx[:half])) + list(reversed(idx[half:])) for i in range(n_flows)]


def flow_inverse(p, pre, z, condition, n_layers, n_group, kernel_size=(3, 3)):
    """Flow.inverse (:515-556) with the incremental row cache of ResidualBlock.add_input (:248-294)."""
    B, _, H, W = z.shape
    dil_h = DILATIONS_H[n_group]
    x = torch.zeros_like(z)
    x[:, :, :1] = z[:, :, :1]
    C = p[pre + "input_proj.weight"].shape[0]
    bufs = [None] * n_layers
    for i in range(1, H):
        x_row = x[:, :, i - 1:i]
        z_row = z[:, :, i:i + 1]
        c_row = condition[:, :, i:i + 1]
        h = F.conv2d(x_row, p[pre + "input_proj.weight"], p[pre + "input_proj.bias"])
        skips = 0
        for l in range(n_layers):
            q = f"{pre}resnet.{l}."
            dil = (dil_h[l], 2 ** l)
            rh = 1 + (kernel_size[0] - 1) * dil[0]
            rw = 1 + (kernel_size[1] - 1) * dil[1]
            if bufs[l] is None:
                bufs[l] = torch.zeros(B, C, rh, W, dtype=z.dtype)
            bufs[l] = torch.cat([bufs[l][:, :, 1:], h], dim=2)
            xin = h
            y = F.conv2d(F.pad(bufs[l], (rw // 2, (rw - 1) // 2, 0, 0)), p[q + "conv.weight"], p[q + "conv.bias"], dilation=dil)
            y = y + F.conv2d(c_row, p[q + "condition_proj.weight"], p[q + "condition_proj.bias"])
            content, gate = torch.chunk(y, 2, dim=1)
            y = torch.tanh(content) * torch.sigmoid(gate)
            y = F.conv2d(y, p[q + "out_proj.weight"], p[q + "out_proj.bias"])
            res, skip = torch.chunk(y, 2, dim=1)
            h = xin + res
            skips = skips + skip
        params = F.conv2d(skips, p[pre + "output_proj.weight"], p[pre + "output_proj.bias"])
        logs, b = torch.chunk(params, 2, dim=1)
        x[:, :, i:i + 1] = (z_row - b) * torch.exp(-logs)
    return x


def waveflow_inverse(p, z, condition, n_flows, n_layers, n_group):
    """WaveFlow.inverse (:674-711): z (B, T), condition (B, C, T) -> x (B, T')."""
    pruned = z.shape[-1] // n_group * n_group
    z, condition = z[:, :pruned], condition[:, :, :pruned]
    B = z.shape[0]
    z = z.reshape(B, -1, n_group).transpose(1, 2).unsqueeze(1)                       # (B, 1, H, W)
    condition = condition.reshape(B, condition.shape[1], -1, n_group).transpose(2, 3)  # (B, C, H, W)
    perms = create_perm(n_group, n_flows)
    for i in reversed(range(n_flows)):
        pi = torch.tensor(perms[i])
        z = z.index_select(2, pi)
        condition = condition.index_select(2, pi)
        z = flow_inverse(p, f"decoder.{i}.", z, condition, n_layers, n_group)
    x = z.squeeze(1)
    return x.transpose(1, 2).reshape(B, -1)


def infer(p, mel, z, n_up=2, n_flows=8, n_layers=8, n_group=16):
    """ConditionalWaveFlow.infer (:784-805) with caller-supplied noise z (B, T_c)."""
    cond = encoder(p, mel, n_up, trim_conv_artifact=True)
    return waveflow_inverse(p, z, cond, n_flows, n_layers, n_group)


def synth_params(seed=4, upsample_factors=(16, 16), n_flows=8, n_layers=8, n_group=16, channels=64, n_mels=80, kernel_size=(3, 3),
                 weight_norm=True):
    g = torch.Generator().manual_seed(seed)
    p = {}

    def u(*shape, std):
        return (torch.rand(*shape, generator=g) * 2 - 1) * std

    for i, f in enumerate(upsample_factors):
        std = math.sqrt(1 / (3 * 2 * f))
        p[f"encoder.{i}.weight"] = u(1, 1, 3, 2 * f, std=std) + 1.0 / (3 * 2)   # positive-ish smoothing kernel
        p[f"encoder.{i}.bias"] = u(1, std=std)
    C = channels
    for fl in range(n_flows):
        pre = f"decoder.{fl}."
        p[pre + "input_proj.weight"] = u(C, 1, 1, 1, std=1.0)
        p[pre + "input_proj.bias"] = u(C, std=1.0)
        for l in range(n_layers):
            q = f"{pre}resnet.{l}."
            std = math.sqrt(1 / (C * kernel_size[0] * kernel_size[1]))
            p[q + "conv.weight"] = u(2 * C, C, *kernel_size, std=std * 1.7)
            p[q + "conv.bias"] = u(2 * C, std=std)
            std = math.sqrt(1 / n_mels)
            p[q + "condition_proj.weight"] = u(2 * C, n_mels, 1, 1, std=std)
            p[q + "condition_proj.bias"] = u(2 * C, std=std)
            std = math.sqrt(1 / C)
            p[q + "out_proj.weight"] = u(2 * C, C, 1, 1, std=std * 1.7)
            p[q + "out_proj.bias"] = u(2 * C, std=std)
        # the reference zero-initialises output_proj (identity flow); use small random values so the test has teeth
        p[pre + "output_proj.weight"] = u(2, C, 1, 1, std=0.05)
        p[pre + "output_proj.bias"] = u(2, std=0.05)
    if weight_norm:
        q = {}
        for k, v in p.items():
            if k.endswith(".weight") and "output_proj" not in k:
                norm = v.reshape(v.shape[0], -1).norm(dim=1)
                q[k + "_g"] = norm * (0.7 + 0.6 * torch.rand(v.shape[0], generator=g))
                q[k + "_v"] = v
            else:
                q[k] = v
        return q
    return p


def flow_forward(p, pre, x, condition, n_layers, n_group, kernel_size=(3, 3)):
    """Flow.forward (:465-494) with the full (non-incremental) ResidualBlock.forward (:209-226): causal padding
    [rh-1, 0] along the height, 'same' along the width.  Used only as the self-consistency check inverse(forward(x)) == x."""
    dil_h = DILATIONS_H[n_group]
    h = F.conv2d(x[:, :, :-1], p[pre + "input_proj.weight"], p[pre + "input_proj.bias"])
    cond = condition[:, :, 1:]
    skips = 0
    for l in range(n_layers):
        q = f"{pre}resnet.{l}."
        dil = (dil_h[l], 2 ** l)
        rh = 1 + (kernel_size[0] - 1) * dil[0]
        rw = 1 + (kernel_size[1] - 1) * dil[1]
        y = F.conv2d(F.pad(h, (rw // 2, (rw - 1) // 2, rh - 1, 0)), p[q + "conv.weight"], p[q + "conv.bias"], dilation=dil)
        y = y + F.conv2d(cond, p[q + "condition_proj.weight"], p[q + "condition_proj.bias"])
        content, gate = torch.chunk(y, 2, dim=1)
        y = torch.tanh(content) * torch.sigmoid(gate)
        y = F.conv2d(y, p[q + "out_proj.weight"], p[q + "out_proj.bias"])
        res, skip = torch.chunk(y, 2, dim=1)
        h = h + res
        skips = skips + skip
    params = F.conv2d(skips, p[pre + "output_proj.weight"], p[pre + "output_proj.bias"])
    logs, b = torch.chunk(params, 2, dim=1)
    z = torch.cat([x[:, :, :1], x[:, :, 1:] * torch.exp(logs) + b], dim=2)   # _transform :456-463
    return z, logs
