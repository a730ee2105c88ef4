"""FP8 decoder projections, checks that need no GPU: the weight quantizer (product and oracle) is bit-identical to
transformers' Fp8Quantize, the oracle's dequantization is Fp8Dequantize, the activation rule is torch's e4m3 conversion,
and the shipped SASS of the FP8 GEMMs is pipelined QGMMA."""
import os

os.environ.setdefault("HF_HUB_OFFLINE", "1")  # FP8Linear's matmul kernel would come from the hub: nothing here may fetch it

import re
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]


class _Cfg:
    weight_block_size = (128, 128)


class _Quantizer:
    quantization_config = _Cfg()


def _hf_convert(w):
    from transformers.integrations.finegrained_fp8 import Fp8Quantize

    out = Fp8Quantize(_Quantizer()).convert({"x.weight": [w]})
    return out["x.weight"], out["x.weight_scale_inv"]


def _weights():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(384, 512, generator=g) * 0.05).to(torch.bfloat16)
    w[128:256, 0:128] = 0                      # an all-zero block: scale 1
    w[0:128, 256:384] *= 3000                  # a large-magnitude block
    w[256:384, 384:512] *= 1e-4                # a tiny-magnitude block
    return w


def test_weight_quantizer_is_hf_fp8quantize():
    from audio_flamingo_b200.modeling import dequantize_fp8_blocks, quantize_fp8_blocks
    from oracle import fp8_oracle as F

    w = _weights()
    q_hf, s_hf = _hf_convert(w)
    for quant in (quantize_fp8_blocks, F.quantize_weight):
        q, s = quant(w)
        assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32 and s.shape == (3, 4)
        assert torch.equal(q.view(torch.uint8), q_hf.view(torch.uint8))
        assert torch.equal(s, s_hf)
    assert s_hf[1, 0].item() == 1.0
    from transformers.integrations.finegrained_fp8 import Fp8Dequantize

    class Q(_Quantizer):
        pass

    deq = Fp8Dequantize(Q()).convert({"weight$": [q_hf], "weight_scale_inv": [s_hf]}, full_layer_name="x.weight")["x.weight"]
    assert torch.equal(F.dequantize_weight(q_hf, s_hf), deq.reshape(w.shape))
    assert torch.equal(dequantize_fp8_blocks(q_hf, s_hf), deq.reshape(w.shape))


def test_weight_quantizer_on_the_tiny_decoder():
    from audio_flamingo_b200.modeling import quantize_fp8_blocks
    from oracle import af3_oracle as O

    sd = O.hf_model("tiny", seed=0).state_dict()
    n = 0
    for k, v in sd.items():
        if k.startswith("language_model.model.layers.") and k.endswith("proj.weight"):
            q_hf, s_hf = _hf_convert(v.to(torch.bfloat16))
            q, s = quantize_fp8_blocks(v.to(torch.bfloat16))
            assert torch.equal(q.view(torch.uint8), q_hf.view(torch.uint8)) and torch.equal(s, s_hf), k
            n += 1
    assert n == 2 * 7


def test_activation_rule_is_torch_e4m3_conversion():
    """q = e4m3(x / s) with s = amax / 448: every |x / s| <= 448 rounds to a finite e4m3 value, and the group maximum maps
    to +-448 exactly."""
    from oracle import fp8_oracle as F

    g = torch.Generator().manual_seed(1)
    x = (torch.randn(9, 512, generator=g) * torch.logspace(-6, 4, 9)[:, None]).to(torch.bfloat16)
    x[3, 128:256] = 0
    q, s = F.quantize_activation(x)
    assert s[3, 1].item() == 1.0 and (q[3, 128:256].float() == 0).all()
    xf = x.float().reshape(9, 4, 128)
    amax = xf.abs().amax(-1)
    s_rule = torch.where(amax > 0, amax / torch.full_like(amax, 448.0), torch.ones_like(amax))
    assert torch.equal(s, s_rule)
    q_rule = (xf / s_rule[..., None]).to(torch.float8_e4m3fn).reshape(9, 512)
    assert torch.equal(q.view(torch.uint8), q_rule.view(torch.uint8))
    qf = q.float().reshape(9, 4, 128)
    assert torch.isfinite(qf).all()
    nz = amax > 0
    assert torch.equal(qf.abs().amax(-1)[nz], torch.full_like(amax[nz], 448.0))


def _sass_functions():
    from audio_flamingo_b200 import _lib, build

    build.build()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.lib_path())], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return funcs


def test_fp8_gemms_issue_pipelined_qgmma():
    """Every kernel with e4m3 warpgroup MMAs (QGMMA) has fewer full waits than QGMMAs: ptxas did not serialise it."""
    funcs = _sass_functions()
    n_kernels = 0
    for name, lines in funcs.items():
        n_mma = sum(1 for l in lines if re.search(r"\bQGMMA\.", l))
        if n_mma == 0:
            continue
        n_kernels += 1
        n_full_wait = sum(1 for l in lines if re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x0\b", l))
        assert n_full_wait < n_mma, f"{name}: {n_full_wait} full wgmma waits for {n_mma} QGMMA"
        assert not any(re.search(r"\bHGMMA\.", l) for l in lines), name
    assert n_kernels >= 5, f"only {n_kernels} kernels with QGMMA"


def test_fp8_symbols_are_exported():
    from audio_flamingo_b200 import _lib

    lib = _lib.load()
    for s in ("af3_quant_fp8", "af3_gemm_fp8", "af3_gemm_qkv_rope_fp8"):
        assert hasattr(lib, s) and s in _lib.SIGNATURES
    # argument validation before any CUDA call
    assert lib.af3_gemm_fp8(None, None, 128, None, None, 128, None, None, 128, 4, 128, 100, 0, None, None, 0, None, 0) != 0
    assert b"multiples of 128" in lib.af3_last_error()
    assert lib.af3_quant_fp8(None, None, 128, None, None, 4, 100) != 0


def test_fp8_load_rejects_sizes_that_are_not_multiples_of_128():
    from audio_flamingo_b200 import AF3Error, AudioFlamingo3ForConditionalGeneration
    from oracle import af3_oracle as O

    p = dict(O.TINY)
    p["text"] = dict(O.TINY["text"], intermediate_size=320)
    ref = O.hf_model(p, seed=0)
    m = AudioFlamingo3ForConditionalGeneration(ref.config)
    with pytest.raises(AF3Error, match="multiples of 128"):
        m.load_reference_state_dict(ref.state_dict(), device="cpu", quantization="fp8")
    with pytest.raises(AF3Error, match="quantization"):
        m.load_reference_state_dict(ref.state_dict(), device="cpu", quantization="int4")


def test_token_major_fp8_gemm_is_warp_specialised_qgmma():
    """The FP8 GEMM above 64 tokens issues m64n128k32 QGMMAs, and its producer warpgroup hands registers to the consumers."""
    funcs = _sass_functions()
    tok = {n: "\n".join(l) for n, l in funcs.items() if "gemm_fp8_tok_kernel" in n}
    assert len(tok) == 4, sorted(tok)
    for name, text in tok.items():
        assert re.search(r"\bQGMMA\.64x128x32\b", text), f"{name}: no m64n128k32 QGMMA"
        assert "USETMAXREG.DEALLOC" in text and "USETMAXREG.TRY_ALLOC" in text, name


def test_fp8_load_rejects_an_e4m3_projection_without_its_scales():
    from audio_flamingo_b200 import AF3Error, AudioFlamingo3ForConditionalGeneration
    from oracle import af3_oracle as O

    ref = O.hf_model("tiny", seed=0)
    sd = dict(ref.state_dict())
    k = "language_model.model.layers.0.mlp.down_proj.weight"
    sd[k] = sd[k].to(torch.float8_e4m3fn)
    m = AudioFlamingo3ForConditionalGeneration(ref.config)
    for q in ("fp8", None):
        with pytest.raises(AF3Error, match="without"):
            m.load_reference_state_dict(sd, device="cpu", quantization=q)
