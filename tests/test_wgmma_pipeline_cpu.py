"""The wgmma pipelines stay asynchronous: in the shipped sm_90a SASS, no kernel waits for every warpgroup MMA to retire
before issuing the next one.

ptxas serialises all wgmma of a kernel (warning C7510: a full `WARPGROUP.DEPBAR.LE gsb0, 0x0` after every HGMMA) when the
kernel contains a function call, e.g. a printf on an error path.  Then each kernel has as many full waits as HGMMAs; with a
k-block group in flight (or several MMAs issued per wait) it has fewer."""
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


def test_no_kernel_serialises_its_wgmma():
    funcs = _sass_functions()
    counted = 0
    for name, lines in funcs.items():
        n_mma = sum(1 for l in lines if re.search(r"\bHGMMA\.", l))
        if n_mma == 0:
            continue
        counted += 1
        n_full_wait = sum(1 for l in lines if re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x0\b", l))
        assert n_full_wait < n_mma, f"{name}: {n_full_wait} full wgmma waits for {n_mma} HGMMA (serialised pipeline)"
    # the GEMMs (both modes), prefill attention and decode attention all issue wgmma
    assert counted >= 4, f"only {counted} kernels with HGMMA found"
    names = " ".join(n for n, l in funcs.items() if any("HGMMA" in x for x in l))
    for kern in ("gemm_tok_kernel", "gemm_kernel", "attention_kernel", "decode_attn_kernel"):
        assert kern in names, kern


def test_normal_mode_gemm_moves_registers_to_the_consumers():
    """The normal-mode GEMM's producer warpgroup hands registers to the two MMA warpgroups (setmaxnreg)."""
    funcs = _sass_functions()
    tok = {n: l for n, l in funcs.items() if "gemm_tok_kernel" in n}
    assert tok
    for name, lines in tok.items():
        text = "\n".join(lines)
        assert "USETMAXREG.DEALLOC" in text and "USETMAXREG.TRY_ALLOC" in text, name
