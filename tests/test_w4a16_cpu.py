"""W4A16 decoder weights without a GPU: the load-time quantizer bit for bit against the format's restatement
(oracle/w4a16_oracle.py) on random weights and every rounding edge, pack / unpack round trips, the load errors, a CPU load
and its state_dict, the C ABI's argument checks, and the SASS of the W4A16 few-token kernels."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

bf16 = torch.bfloat16


def _edge_weight():
    """8 rows x 256 columns (two groups per row), each row an edge of the rule."""
    w = torch.randn(8, 256, generator=torch.Generator().manual_seed(5)) * 0.03
    w[0, :128] = 0                                                     # all-zero group: s = 1, q = 0
    w[1, :128] = torch.linspace(-1, 1, 128)                            # values exactly at +-amax
    w[2, :128] = 0
    w[2, :8] = torch.tensor([7.5, 0.5, 1.5, 2.5, -0.5, -2.5, 3.5, -3.5])  # s = bf16(1.0): every x / s is a tie at .5
    w[3, :128] = -7.5                                                  # negative extreme: -7.5 -> -8 (half to even)
    w[3, 5] = 7.5                                                      # positive extreme: +7.5 -> +8, clamped to 7
    w[4, 128:] = 1e-30                                                 # tiny group
    w[5, :128] = 3e4                                                   # large group
    return w.to(bf16)


def test_quantizer_matches_the_restatement_bit_for_bit():
    from audio_flamingo_b200.modeling import quantize_w4a16
    from oracle import w4a16_oracle as W

    for w in (_edge_weight(), (torch.randn(384, 1024, generator=torch.Generator().manual_seed(1)) * 0.02).to(bf16),
              (torch.randn(128, 640, generator=torch.Generator().manual_seed(2)) * torch.logspace(-4, 2, 640)).to(bf16)):
        p, s = quantize_w4a16(w)
        pr, sr = W.quantize(w)
        assert p.dtype == torch.int32 and s.dtype == bf16
        assert p.shape == (w.shape[0], w.shape[1] // 8) and s.shape == (w.shape[0], w.shape[1] // 128)
        assert torch.equal(p, pr)
        assert torch.equal(s.view(torch.int16), sr.view(torch.int16))


def test_edge_cases_take_the_specified_codes():
    from audio_flamingo_b200.modeling import quantize_w4a16
    from oracle import w4a16_oracle as W

    p, s = quantize_w4a16(_edge_weight())
    q = W.unpack(p)
    assert s[0, 0].item() == 1.0 and (q[0, :128] == 0).all()
    t = 1.0 / s[1, 0].float()                                           # +-amax / bf16(amax / 7.5): 7.5 give or take the rounding
    assert q[1, 127].item() == min(7, int(torch.round(t))) and q[1, 0].item() == max(-8, int(torch.round(-t)))
    assert s[2, 0].item() == 1.0
    assert q[2, :8].tolist() == [7, 0, 2, 2, 0, -2, 4, -4]              # 7.5 -> 8 -> 7; .5 ties to even
    assert q[3, 0].item() == -8 and q[3, 5].item() == 7
    assert s[4, 1].item() > 0 and q[4, 128:].abs().max().item() <= 8


def test_pack_unpack_round_trips():
    from audio_flamingo_b200.modeling import dequantize_w4a16, quantize_w4a16
    from oracle import w4a16_oracle as W

    w = (torch.randn(256, 512, generator=torch.Generator().manual_seed(3)) * 0.05).to(bf16)
    p, s = quantize_w4a16(w)
    q = W.unpack(p)
    assert int(q.min()) >= -8 and int(q.max()) <= 7
    wd = dequantize_w4a16(p, s)
    assert wd.dtype == bf16 and torch.equal(wd, W.dequantize(p, s))
    assert torch.equal(wd, (q.to(bf16) * s.repeat_interleave(128, 1)))
    # every 4-bit code survives packing: a row holding -8 .. 7 in order
    codes = torch.arange(-8, 8, dtype=torch.float32).repeat(8).reshape(1, 128)
    pc, sc = quantize_w4a16(codes.clamp(min=-7.5).to(bf16))             # amax 7.5 -> s = 1; -7.5 ties to -8
    assert sc.item() == 1.0 and W.unpack(pc).tolist() == codes.to(torch.int64).tolist()


def _tiny(**text):
    from oracle import af3_oracle as O

    p = dict(O.TINY)
    p["text"] = dict(O.TINY["text"], **text)
    return O.hf_model(p, seed=0)


def test_load_errors_are_raised_before_any_cuda_call():
    from audio_flamingo_b200 import AF3Error, AudioFlamingo3ForConditionalGeneration

    ref = _tiny(intermediate_size=320)
    m = AudioFlamingo3ForConditionalGeneration(ref.config)
    with pytest.raises(AF3Error, match="multiples of 128"):
        m.load_reference_state_dict(ref.state_dict(), device="cuda", quantization="w4a16")
    with pytest.raises(AF3Error, match="quantization"):
        m.load_reference_state_dict(ref.state_dict(), device="cuda", quantization="int8")
    ref = _tiny()
    sd = dict(ref.state_dict())
    base = "language_model.model.layers.1.self_attn.o_proj"
    from audio_flamingo_b200.modeling import quantize_w4a16

    p, _ = quantize_w4a16(sd.pop(base + ".weight").to(bf16))
    sd[base + ".weight_packed"] = p
    m = AudioFlamingo3ForConditionalGeneration(ref.config)
    for q in ("w4a16", None, "fp8"):
        with pytest.raises(AF3Error, match="without"):
            m.load_reference_state_dict(sd, device="cuda", quantization=q)


def test_cpu_load_stores_the_packed_format_and_round_trips():
    """A W4A16 load holds weight_packed / weight_scale (the restatement's values) instead of weight on every decoder
    projection, and nothing else changes; its state_dict loads back as W4A16 without the argument, and so does one quantized
    by the restatement."""
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration
    from audio_flamingo_b200.modeling import DECODER_PROJECTIONS
    from oracle import w4a16_oracle as W

    ref = _tiny()
    rsd = ref.state_dict()
    m = AudioFlamingo3ForConditionalGeneration.from_reference(ref, device="cpu", quantization="w4a16")
    assert m.quantization == "w4a16"
    sd = m.state_dict()
    n = 0
    for k, v in rsd.items():
        base = k[: -len(".weight")]
        if k.startswith("language_model.model.layers.") and any(base.endswith(p) for p in DECODER_PROJECTIONS) and k.endswith(".weight"):
            assert k not in sd
            pr, sr = W.quantize(v.to(bf16))
            assert torch.equal(sd[base + ".weight_packed"], pr) and torch.equal(sd[base + ".weight_scale"], sr), base
            n += 1
        else:
            assert torch.equal(sd[k], v.to(bf16) if v.is_floating_point() else v), k
    assert n == 7 * len(m.language_model.model.layers)
    again = AudioFlamingo3ForConditionalGeneration(ref.config)
    again.load_reference_state_dict({k: v.clone() for k, v in sd.items()}, device="cpu")
    assert again.quantization == "w4a16"
    assert all(torch.equal(v, sd[k]) for k, v in again.state_dict().items())
    # back to bf16 in place: the module tree gets its weights back
    again.load_reference_state_dict(rsd, device="cpu")
    assert again.quantization is None
    assert sorted(again.state_dict()) == sorted(rsd)


def test_symbols_and_argument_checks_without_a_device():
    from audio_flamingo_b200 import _lib

    header = (Path(__file__).resolve().parents[1] / "include" / "af3b200.h").read_text()
    lib = _lib.load()
    for s in ("af3_gemm_w4a16", "af3_gemm_qkv_rope_w4a16", "af3_dequant_w4a16"):
        assert hasattr(lib, s) and s in _lib.SIGNATURES and re.search(rf"\b{s}\(", header), s
    assert lib.af3_abi_version() == 4
    # n_tok above 64: the error names the limit
    assert lib.af3_gemm_w4a16(None, None, 128, None, 16, None, 1, None, 128, 65, 128, 128, 0, None, None, 0, None, 0) != 0
    assert b"64" in lib.af3_last_error()
    assert lib.af3_gemm_w4a16(None, None, 128, None, 16, None, 1, None, 128, 4, 128, 100, 0, None, None, 0, None, 0) != 0
    assert b"multiples of 128" in lib.af3_last_error()
    assert lib.af3_dequant_w4a16(None, None, 16, None, 1, None, 4, 100) != 0
    assert b"multiples of 128" in lib.af3_last_error() or b"multiple of 128" in lib.af3_last_error()
    assert lib.af3_gemm_qkv_rope_w4a16(None, None, 128, None, 16, None, 1, None, None, 128, 4, 128, 28, 4, 64, None, None, None, 16,
                                       None, None, 0) != 0
    assert b"head_dim" in lib.af3_last_error()


def test_w4a16_kernels_issue_register_a_hgmma_without_local_memory():
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
    # gemm_kernel<BN, NA, STAGES, EPI, WM_W4 = 2>
    w4 = {n: l for n, l in funcs.items() if re.match(r"_ZN3af311gemm_kernelILi32ELi[12]ELi\d+ELi\d+ELi2EEEv", n)}
    assert len(w4) == 5, sorted(w4)
    for n, lines in w4.items():
        mma = [l for l in lines if re.search(r"\bHGMMA\.64x32x16\.F32\.BF16\b", l)]
        assert mma and all(re.search(r"HGMMA\.\S+ R\d+, R\d+, gdesc\[", l) for l in mma), f"{n}: A must come from registers"
        assert not any(re.search(r"\b(LDL|STL)\b", l) for l in lines), f"{n}: local memory"
