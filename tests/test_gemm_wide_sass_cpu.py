"""The wide normal-mode GEMM that the prefill shapes take is built as intended: in the shipped sm_90a SASS it issues
m64n256 warpgroup MMAs (one weight slice per k16 step, shared by both consumer warpgroups) and nothing narrower, and its
producer warpgroup hands its registers to the consumers."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest


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


def test_wide_gemm_issues_m64n256():
    funcs = _sass_functions()
    wide = {n: "\n".join(l) for n, l in funcs.items() if "gemm_tok_wide_kernel" in n}
    assert wide, "no wide normal-mode GEMM in the library"
    for name, text in wide.items():
        assert re.search(r"\bHGMMA\.64x256x16\b", text), f"{name}: no m64n256k16 wgmma"
        assert not re.search(r"\bHGMMA\.64x128x16\b", text), f"{name}: narrower wgmma in the wide kernel"
        assert "USETMAXREG.DEALLOC" in text and "USETMAXREG.TRY_ALLOC" in text, name
