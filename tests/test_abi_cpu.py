"""C-ABI checks that need no GPU: the library builds/loads, exports every symbol include/af3b200.h declares, the
ctypes table covers the header one to one, and the product path fails loudly (no CPU fallback)."""
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def lib():
    from audio_flamingo_b200 import _lib, build

    build.build()
    return _lib.load()


def _header_symbols():
    text = (ROOT / "include" / "af3b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(af3_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported(lib):
    from audio_flamingo_b200 import _lib

    syms = _header_symbols()
    assert len(syms) >= 16
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in af3b200.h but not exported"
    assert sorted(_lib.SIGNATURES) == syms, "ctypes signature table and header disagree"
    assert lib.af3_abi_version() == 4   # v2: trace API; v3: af3_gated_residual, af3_token_step; v4: RMSNorm fusion removed


def test_library_contains_hopper_instructions():
    """The shipped .so carries sm_90a SASS with warpgroup MMA (HGMMA) and TMA (UTMALDG)."""
    import shutil
    import subprocess

    from audio_flamingo_b200 import _lib

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.lib_path())], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnem in ("HGMMA", "UTMALDG"):
        assert mnem in sass, mnem


def test_error_reporting_without_gpu(lib):
    # argument validation happens before any CUDA call: non-zero status + message through af3_last_error
    rc = lib.af3_gemm_bf16(None, None, 8, None, 8, None, 8, 0, 16, 64, 0, None, None, 0, 0)
    assert rc != 0
    assert b"gemm" in lib.af3_last_error()
    rc = lib.af3_attention(None, None, 0, None, None, 0, 0, 0, None, 8, 1, 3, 2, 64, 4, 4, 1.0, 0, None, None)
    assert rc != 0 and b"multiple of Hkv" in lib.af3_last_error()


def test_no_cpu_fallback():
    from audio_flamingo_b200 import AF3Error, ops

    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    with pytest.raises(AF3Error, match="CUDA"):
        ops.linear(x, x)
    with pytest.raises(AF3Error, match="CUDA"):
        ops.layernorm(x, x[0], x[0])


def test_product_does_not_import_oracle():
    for p in (ROOT / "audio_flamingo_b200").rglob("*.py"):
        assert "oracle" not in p.read_text().replace("the oracle", ""), f"{p} references the oracle"
