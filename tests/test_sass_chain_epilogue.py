"""SASS of the layer-chain kernels in the built library (no GPU needed): the epilogue splits each value into its bf16
hi/lo pair once, writes the pairs into the operand buffer with stmatrix, and the bf16 images leave by TMA store.

Per layer body (NB = 1, 2) the rolled epilogue converts one 16-value group: 8 bf16x2 conversions for the hi words, 8 more
for the lo words with two planes.  A second split of the same values (the old separate image store) doubles the count."""
import os
import re
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(REPO, "dsac-v2_b200", "libdsact.so")


def _cuobjdump():
    for d in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", "cuobjdump")):
            return os.path.join(d, "bin", "cuobjdump")
    return shutil.which("cuobjdump")


@pytest.fixture(scope="module")
def chain_sass():
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built libdsact.so and the CUDA toolkit's cuobjdump")
    text = subprocess.run([tool, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", text)[1:]:
        name, body = chunk.split("\n", 1)
        if "tc_chain_kernel" in name:
            funcs[name.strip()] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
    assert len(funcs) == 4, sorted(funcs)
    return funcs


def _count(ins, op):
    return sum(1 for s in ins if re.search(r"(^|\s)" + op + r"(\.|\s|$)", s))


def test_operand_buffer_written_by_stmatrix_and_images_by_tma_store(chain_sass):
    for name, ins in chain_sass.items():
        assert _count(ins, "STSM") > 0, f"{name}: no STSM"
        assert _count(ins, "UTMASTG") > 0, f"{name}: no UTMASTG"


def test_each_value_is_split_once(chain_sass):
    for name, ins in chain_sass.items():
        planes2 = re.search(r"tc_chain_kernelILb([01])E", name).group(1) == "1"
        assert _count(ins, "F2FP") == (32 if planes2 else 16), (name, _count(ins, "F2FP"))
