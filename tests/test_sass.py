"""SASS of the tensor-core kernels in the built library (no GPU needed): the wgmma.mma_async of one k-block issue back to
back, and one k-block of them stays in flight while the next is issued.

ptxas serialises wgmma when the accumulator registers are touched on a path it cannot prove warp-uniform (C7520: it
then waits for every MMA to retire before the next one issues).  It reports that only under -Xptxas -v, and the
results stay the same, so nothing but the instruction stream shows the regression."""
import os
import re
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(REPO, "dsac-v2_b200", "libdsact.so")
KERNELS = ("tc_chain_kernel", "tc_gemm_kernel")


def _cuobjdump():
    for d in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", "cuobjdump")):
            return os.path.join(d, "bin", "cuobjdump")
    return shutil.which("cuobjdump")


@pytest.fixture(scope="module")
def sass():
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built libdsact.so and the CUDA toolkit's cuobjdump")
    text = subprocess.run([tool, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", text)[1:]:
        name, body = chunk.split("\n", 1)
        if any(k in name for k in KERNELS):
            funcs[name.strip()] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
    return funcs


def test_every_tensor_core_kernel_is_present(sass):
    # 2 plane counts x 2 B orientations of the chain kernel, 2 plane counts x 3 orientations of the GEMM kernel
    assert sum("tc_chain_kernel" in n for n in sass) == 4, sorted(sass)
    assert sum("tc_gemm_kernel" in n for n in sass) == 6, sorted(sass)


def test_no_full_wait_between_the_mmas_of_a_k_block(sass):
    # Between one HGMMA and the next, a full wait (WARPGROUP.DEPBAR.LE gsb0, 0x0) is only allowed where a new k-block
    # begins, that is after the mbarrier wait on its ring slot (SYNCS.PHASECHK).
    bad = {}
    for name, ins in sass.items():
        hg = [i for i, s in enumerate(ins) if s.startswith("HGMMA") or " HGMMA" in s]
        assert hg, f"{name}: no HGMMA"
        n = 0
        for a, b in zip(hg, hg[1:]):
            between = ins[a + 1:b]
            if any("DEPBAR.LE gsb0, 0x0" in s for s in between) and not any("SYNCS.PHASECHK" in s for s in between):
                n += 1
        if n:
            bad[name] = f"{n} of {len(hg)} HGMMAs wait for all MMAs before the next one issues"
    assert not bad, bad


def test_one_k_block_stays_in_flight(sass):
    # after a k-block is issued, only the one before it is waited for
    for name, ins in sass.items():
        assert any("DEPBAR.LE gsb0, 0x1" in s for s in ins), f"{name}: no wgmma.wait_group 1"
