"""CPU tests: the C-ABI library loads and exports everything the header declares; host-side logic."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from parakeet_b200 import _lib, ops


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    names = _lib.exported_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/parakeet_b200.h but not exported"
    assert L.pk_version() >= 100
    assert isinstance(L.pk_last_error(), bytes)


def test_bad_arguments_return_error_codes_not_crashes():
    L = _lib.lib()
    rc = L.pk_split_f32(None, None, None, 10, None)
    assert rc == -1 and b"NULL" in L.pk_last_error()
    args = _lib.ConvGemmArgs()
    assert L.pk_conv_gemm(ctypes.byref(args), None) == -1
    assert L.pk_length_regulate(None, None, 1, 1, 1, 1, None, None, None, None) == -1


def test_no_cpu_fallback():
    with pytest.raises(_lib.PkError):
        ops.Split.from_f32(torch.zeros(4, 4))
    from parakeet_b200.models import FastSpeech2, PWGGenerator
    m = FastSpeech2(20, 80, adim=64, aheads=1, elayers=1, dlayers=1, eunits=64, dunits=64, postnet_chans=64, device="cpu")
    with pytest.raises(_lib.PkError):
        m.inference(torch.tensor([1, 2, 3]))
    g = PWGGenerator(layers=3, stacks=1, device="cpu")
    with pytest.raises(_lib.PkError):
        g(torch.zeros(1, 1, 256), torch.zeros(1, 80, 5))


def test_pack_weight_layout():
    w = torch.arange(2 * 80 * 3, dtype=torch.float32).reshape(2, 80, 3)
    p = ops.pack_weight(w, device="cpu")
    assert list(p.hi.shape) == [2, 3 * 128]
    full = p.float()
    for tap in range(3):
        assert torch.allclose(full[:, tap * 128:tap * 128 + 80], w[:, :, tap], rtol=2 ** -15)
        assert full[:, tap * 128 + 80:(tap + 1) * 128].abs().max() == 0


def test_state_dict_keys_match_reference_names():
    from parakeet_b200.models import FastSpeech2, PWGGenerator
    from oracle import fastspeech2 as ofs
    from oracle import pwg as opwg
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, device="cpu")
    assert set(m.state_dict()) == set(ofs.synth_params(1))
    assert tuple(m.state_dict()["encoder.encoders.0.self_attn.linear_q.weight"].shape) == (384, 384)
    assert tuple(m.state_dict()["encoder.encoders.0.feed_forward.w_1.weight"].shape) == (1536, 384, 3)
    assert tuple(m.state_dict()["postnet.postnet.0.1._variance"].shape) == (256,)
    g = PWGGenerator(**opwg.DEFAULT_GENERATOR_PARAMS, device="cpu")
    assert set(g.state_dict()) == set(opwg.synth_params(2, weight_norm=True))
    assert g.state_dict()["conv_layers.0.conv.weight_g"].dim() == 1
    g.remove_weight_norm()
    assert set(g.state_dict()) == set(opwg.synth_params(2))
    with pytest.raises(KeyError):
        g.set_state_dict({})


def test_weight_norm_roundtrip_matches_oracle_fold():
    from parakeet_b200.models import PWGGenerator
    from oracle import pwg as opwg
    g = PWGGenerator(**opwg.DEFAULT_GENERATOR_PARAMS, device="cpu")
    pw = opwg.synth_params(2, weight_norm=True)
    g.set_state_dict(pw)
    g.remove_weight_norm()
    ref = opwg.fold_weight_norm(pw)
    for k, v in g.state_dict().items():
        assert torch.allclose(v, ref[k], rtol=1e-6, atol=1e-7), k


def test_polyphase_table_equals_stretch_then_fir():
    # the identity behind pk_pwg_upsample: nearest stretch by s + FIR(2s+1, zero pad s) == 3-tap polyphase filter
    rng = np.random.default_rng(0)
    for s in (3, 4, 5):
        w = rng.standard_normal(2 * s + 1).astype(np.float32)
        x = rng.standard_normal(11).astype(np.float32)
        u = np.repeat(x, s)
        ref = np.convolve(np.pad(u, (s, s)), w[::-1], mode="valid")
        poly = np.zeros((3, s), np.float32)
        for r in range(s):
            for q in range(2 * s + 1):
                poly[(r + q) // s, r] += w[q]
        xp = np.pad(x, (1, 1))
        out = np.array([sum(poly[k, t % s] * xp[t // s + k] for k in range(3)) for t in range(s * len(x))])
        assert np.allclose(out, ref, atol=1e-5)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gcc():
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    return gcc


def test_header_is_plain_c_and_struct_layouts_match_ctypes(tmp_path):
    """include/parakeet_b200.h must compile as C (it is what a cgo / ctypes / cffi binding consumes) and every struct it declares
    must be bound by parakeet_b200/_lib.py, under its mechanical class name, with the C compiler's field offsets and sizes."""
    gcc = _gcc()
    mirrors = _lib.STRUCTS
    # the parse misses no struct: count the `struct` keywords of the header with its comments stripped by the compiler
    bare = subprocess.run([gcc, "-fpreprocessed", "-dD", "-E", "-P", os.path.join(ROOT, "include", "parakeet_b200.h")],
                          check=True, capture_output=True, text=True).stdout
    assert len(re.findall(r"\bstruct\b", bare)) == len(mirrors)
    names = {"pk_operand": "Operand", "pk_conv_gemm_args": "ConvGemmArgs", "pk_gemm_epilogue": "GemmEpilogue",
             "pk_pwg_layer_args": "PwgLayerArgs", "pk_pwg_layer_fc_args": "PwgLayerFcArgs", "PkAttentionArgs": "AttentionArgs",
             "pk_waveflow_flow_args": "WaveflowFlowArgs",
             "pk_waveflow_forward_layer_args": "WaveflowForwardLayerArgs", "pk_waveflow_forward_tail_args": "WaveflowForwardTailArgs",
             "pk_ss_residual_block_args": "SsResidualBlockArgs", "pk_waveflow_backward_layer_args": "WaveflowBackwardLayerArgs",
             "PkTaco2DecodeArgs": "Taco2DecodeArgs", "PkTtsDecodeArgs": "TtsDecodeArgs"}
    for cname, pyname in names.items():
        assert mirrors[cname] is getattr(_lib, pyname), (cname, pyname)
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "parakeet_b200.h"', "int main(void) {"]
    for cname, cls in mirrors.items():
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    seen = 0
    for line in out.splitlines():
        cname, field, value = line.split()
        cls = mirrors[cname]
        expect = ctypes.sizeof(cls) if field == "size" else getattr(cls, field).offset
        assert int(value) == expect, (cname, field, value, expect)
        seen += 1
    assert seen == sum(len(c._fields_) + 1 for c in mirrors.values())


_C_NAMES = {ctypes.c_int32: "int32_t", ctypes.c_int64: "int64_t", ctypes.c_uint32: "uint32_t", ctypes.c_uint64: "uint64_t",
            ctypes.c_float: "float", ctypes.c_char_p: "const char*"}


def test_bound_signatures_match_the_header(tmp_path):
    """Every entry point's restype and argtypes, as lib() binds them, are rebuilt as a C function pointer type to which the
    header's function must be assignable under -Werror: a missing, extra or differently typed parameter or return fails to
    compile.  ctypes binds every pointer as a pointer, so a bound pointer is rebuilt with the header's spelling at its
    position when the header has a pointer there, and as void* (which no scalar accepts) when it has not."""
    gcc = _gcc()
    L = _lib.lib()
    lines = ['#include "parakeet_b200.h"']
    for name, proto in _lib.PROTOTYPES.items():
        fn = getattr(L, name)
        spelled = [re.sub(r"\s*\w+$", "", p) for p in proto.params]        # the header's types without parameter names
        params = []
        for i, t in enumerate(fn.argtypes or []):
            if t is ctypes.c_void_p or issubclass(t, ctypes._Pointer):
                is_ptr = i < len(spelled) and ("*" in spelled[i] or spelled[i] == "pk_stream_t")
                params.append(spelled[i] if is_ptr else "void*")
            else:
                params.append(_C_NAMES[t])
        lines.append(f"{_C_NAMES[fn.restype]} (*fp_{name})({', '.join(params) or 'void'}) = {name};")
    src = tmp_path / "signatures.c"
    src.write_text("\n".join(lines) + "\n")
    r = subprocess.run([gcc, "-std=c99", "-Werror", "-Wincompatible-pointer-types", "-I", os.path.join(ROOT, "include"), "-c",
                        str(src), "-o", str(tmp_path / "signatures.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert len(_lib.PROTOTYPES) == len(_lib.exported_symbols()) >= 100


def test_header_parse_refuses_unknown_types():
    with pytest.raises(_lib.PkError, match="pk_x"):
        _lib.parse_header("typedef void* pk_stream_t;\nint pk_x(size_t n, pk_stream_t stream);\n")
    with pytest.raises(_lib.PkError, match="pk_y_args"):
        _lib.parse_header("typedef struct pk_y_args { int32_t n; double scale; } pk_y_args;\n")
    with pytest.raises(_lib.PkError, match="pk_z"):
        _lib.parse_header("size_t pk_z(void);\n")
