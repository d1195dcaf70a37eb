"""The build refuses objects in which ptxas serialized a wgmma pipeline (C7510): a function call reachable while a
wgmma group is in flight makes every MMA of the kernel wait for the previous one, silently."""
import os
import shutil

import pytest

from whisperlivekit_b200 import build

LOG = """\
ptxas info    : Compiling entry function '_Z1kPf' for 'sm_90a'
ptxas info    : (C7510) Potential Performance Loss: wgmma.mma_async instructions are serialized due to wgmma pipeline crossing function boundary at a function call in the function '_Z1kPf'
ptxas info    : Used 80 registers, used 1 barriers
"""

# One m64n32k16 wgmma group with a bounded mbarrier wait inside it: with the printf form of the wait ptxas must
# serialize the pipeline, with the trap-only form it must not.
KERNEL = r"""
#include <cstdio>
#include "ptx.cuh"
__global__ void probe(float* out, uint64_t da, uint64_t db, uint32_t bar) {
    float d[16];
    for (int i = 0; i < 16; ++i) d[i] = 0.f;
    wlk::ptx::wgmma_fence();
    wlk::ptx::WgmmaSS<32>::mma(d, da, db, 0u);
    wlk::ptx::wgmma_commit();
    wlk::ptx::WAIT(bar, 0);
    wlk::ptx::wgmma_wait<0>();
    wlk::ptx::wgmma_fence_regs(d);
    for (int i = 0; i < 16; ++i) out[16 * threadIdx.x + i] = d[i];
}
"""


def test_serialized_wgmma_lines():
    assert build.serialized_wgmma(LOG) == [LOG.splitlines()[1].strip()]
    assert build.serialized_wgmma(LOG.replace("(C7510) ", "")) == []
    assert build.serialized_wgmma("") == []


def _nvcc_or_skip():
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    if not os.path.isabs(nvcc) and shutil.which(nvcc) is None:
        pytest.skip("nvcc not found")
    return nvcc


@pytest.mark.parametrize("wait,serialized", [("mbar_wait", True), ("mbar_wait_mma", False)])
def test_compile_object_rejects_serialized_wgmma(tmp_path, wait, serialized):
    nvcc = _nvcc_or_skip()
    src = tmp_path / "probe.cu"
    src.write_text(KERNEL.replace("WAIT", wait))
    obj = tmp_path / "probe.o"
    if serialized:
        with pytest.raises(RuntimeError, match="C7510"):
            build.compile_object(str(src), str(obj), nvcc=nvcc, extra_flags=["-I", build.CSRC])
        assert not obj.exists()          # nothing left behind that a later build would take as up to date
    else:
        build.compile_object(str(src), str(obj), nvcc=nvcc, extra_flags=["-I", build.CSRC])
        assert obj.exists()
