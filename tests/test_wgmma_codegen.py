"""CPU: what ptxas makes of the tensor-core GEMM template (te_tc_wgmma.cu) at the library's build flags.

Every wg_kernel instantiation must compile without a compiler-injected warpgroup.wait (ptxas C7517: a wgmma.wait_group 0
the source did not ask for, which retires every k-block's wgmmas before the next one is issued and so takes away the
k-block the TMA mainloop keeps in flight) and without spills.  Needs nvcc only, no GPU.
"""
import os
import re
import subprocess
import tempfile

import pytest

from transformer_explainability_b200 import build

SRC = os.path.join(build.CSRC, "te_tc_wgmma.cu")

pytestmark = pytest.mark.skipif(not build.have_nvcc(), reason="nvcc not available")


@pytest.fixture(scope="module")
def ptxas_log():
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.CSRC, "-c", SRC,
                                                     "-o", os.path.join(tmp, "te_tc_wgmma.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


def wg_kernels(log):
    """{mangled wg_kernel name: (spill store bytes, spill load bytes)}"""
    out = {}
    for m in re.finditer(r"Function properties for (\S*wg_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", log):
        out[m.group(1)] = (int(m.group(3)), int(m.group(4)))
    return out


def test_every_instantiation_was_found(ptxas_log):
    kernels = wg_kernels(ptxas_log)
    # the z+ rule, layers_lrp, Linear and attention problems: dozens of instantiations
    assert len(kernels) >= 30, sorted(kernels)
    assert any("ZrProb" in k for k in kernels) and any("LinProb" in k for k in kernels)


def test_no_injected_warpgroup_wait(ptxas_log):
    injected = sorted(set(re.findall(r"\(C7517\).*?function '(\S+)'", ptxas_log)))
    assert not [k for k in injected if "wg_kernel" in k], "ptxas injected warpgroup.wait into:\n" + "\n".join(injected)


def test_no_spills(ptxas_log):
    spilled = {k: v for k, v in wg_kernels(ptxas_log).items() if v != (0, 0)}
    assert not spilled, spilled
