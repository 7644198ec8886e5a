"""SASS checks of the wgmma kernels' main loops (no GPU needed: cuobjdump reads the cross-compiled library).

A consumer hands a ring slot back to the producer (of its own CTA or of the peer CTA of a 2-CTA cluster) once its
wgmma reads of the slot have retired.  That release needs no memory fence: the consumer wrote nothing the producer
must see, and the next writer of the slot is a TMA load ordered by the barrier phase.  A `.release.cluster` arrive
nevertheless lowers to MEMBAR.ALL.GPU + ERRBAR + CGAERRBAR, a GPU-wide fence in every consumer warp and every k-block
that stalls the issue of the next wgmma group.  These tests keep such fences out of the main loops."""

import os
import re
import shutil
import subprocess

import pytest

# the main loop: from the function's first HGMMA through the first SYNCS.ARRIVE (the release of the last slot) after
# its last `wgmma.wait_group 0`
_FENCE = re.compile(r"\b(MEMBAR\.ALL\.GPU|MEMBAR\.ALL\.SYS|MEMBAR\.SC\.\w+|ERRBAR|CGAERRBAR)\b")
_FUNC = re.compile(r"^\s*Function : (\S+)")
_INSN = re.compile(r"/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;")


@pytest.fixture(scope="module")
def sass_functions(native_lib):
    """mangled name -> list of SASS instructions of every kernel in the built library"""
    from sonar_b200 import _lib

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    r = subprocess.run([cuobjdump, "-sass", str(_lib.lib_path())], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    funcs, cur = {}, None
    for line in r.stdout.splitlines():
        m = _FUNC.match(line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = _INSN.search(line)
        if m and cur is not None:
            cur.append(m.group(1))
    return funcs


def _main_loop(insns):
    first = next(i for i, s in enumerate(insns) if "HGMMA" in s)
    last_wait = max(i for i, s in enumerate(insns) if "WARPGROUP.DEPBAR.LE gsb0, 0x0" in s)
    end = next(i for i in range(last_wait, len(insns)) if "SYNCS.ARRIVE" in insns[i])
    return insns[first:end + 1]


@pytest.mark.parametrize("kernel", ["gemm_bf16_wgmma_kernel", "attention_tc_kernel", "attention_relpos_tc_kernel"])
def test_no_gpu_scope_fence_in_wgmma_main_loop(sass_functions, kernel):
    mangled = f"{len(kernel)}{kernel}"  # the Itanium-mangled identifier, so that one name is not a prefix of another
    insts = {name: insns for name, insns in sass_functions.items() if mangled in name}
    assert insts, f"no {kernel} in the library"
    fenced = {}
    for name, insns in insts.items():
        found = [s for s in _main_loop(insns) if _FENCE.search(s)]
        if found:
            fenced[name] = found
    assert not fenced, f"fences in the main loop of {len(fenced)} of {len(insts)} {kernel} instantiations: {fenced}"
