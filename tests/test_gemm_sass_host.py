"""The GEMM k-loops release their ring slots without a GPU-scope fence (no GPU needed: reads the SASS of the built library).

Each consumer warpgroup frees a ring slot once `wgmma.wait_group` shows the slot's MMAs complete, by arriving on the slot's `empty` barrier
in every CTA of the cluster.  Written as `mbarrier.arrive.release.cluster`, that arrive compiles to MEMBAR.ALL.CTA + MEMBAR.ALL.GPU in front
of every SYNCS.ARRIVE, once per k-block, and the warpgroup's next `.sync.aligned` wgmma waits for the fences.  The release window checked
here runs from each wgmma wait (WARPGROUP.DEPBAR.LE gsb0) through the barrier arrives that follow it, up to the next MMA issue, named
barrier or exit.  The fences that do publish generic-proxy data lie outside every such window: the `acc_free` arrive after an epilogue
(behind the epilogue's BAR.SYNC), `mlp_fused_kernel`'s and `gemm_ln_kernel`'s grid barriers, and the cluster barrier at kernel exit."""
import os
import re
import shutil
import subprocess

import pytest

GEMM_KERNELS = re.compile(r"gemm_wgmma_kernel|gemm_frag_kernel|gemm_fp8_kernel|mlp_fused_kernel|gemm_ln_kernel")
WINDOW_END = re.compile(r"WARPGROUP\.ARRIVE|WARPGROUP\.DEPBAR|BAR\.SYNC|EXIT")


def _cuobjdump():
    from ezaudio_b200 import build
    for c in (os.path.join(os.path.dirname(build.NVCC), "cuobjdump"), shutil.which("cuobjdump")):
        if c and os.path.exists(c):
            return c
    return None


@pytest.fixture(scope="module")
def gemm_sass():
    """{mangled kernel name: SASS lines} of every GEMM kernel in libezb200.so (built first if missing or older than its sources)."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    from ezaudio_b200 import build
    lib = build.build()
    out = subprocess.run([tool, "-sass", lib], capture_output=True, text=True, check=True).stdout
    kernels = {}
    for f in re.split(r"\n\s*Function : ", out)[1:]:
        name, body = f.split("\n", 1)
        if GEMM_KERNELS.search(name):
            kernels[name.strip()] = body.split("\n")
    return kernels


def release_windows(lines):
    """Instruction runs from each wgmma wait through the last barrier arrive before the next MMA issue / wgmma wait / BAR.SYNC / EXIT."""
    for i, line in enumerate(lines):
        if "WARPGROUP.DEPBAR.LE gsb0" not in line:
            continue
        end = None
        for j in range(i + 1, len(lines)):
            if WINDOW_END.search(lines[j]):
                break
            if "SYNCS.ARRIVE" in lines[j]:
                end = j
        if end is not None:
            yield lines[i:end + 1]


def test_every_gemm_kernel_has_a_slot_release(gemm_sass):
    """The window finder sees what the next test checks: every GEMM kernel releases its slots after a wgmma wait, and the cluster
    kernels do it with remote (SYNCS.ARRIVE.TRANS64.RED) arrives."""
    assert len(gemm_sass) >= 10, sorted(gemm_sass)
    remote = 0
    for name, lines in gemm_sass.items():
        ws = list(release_windows(lines))
        assert ws, f"{name}: no barrier arrive after any wgmma wait"
        remote += any("SYNCS.ARRIVE.TRANS64.RED" in l for w in ws for l in w)
    assert remote >= 10, remote


def test_gemm_slot_release_has_no_gpu_fence(gemm_sass):
    fenced = {}
    for name, lines in gemm_sass.items():
        n = sum(any("MEMBAR.ALL.GPU" in l for l in w) for w in release_windows(lines))
        if n:
            fenced[name] = n
    assert not fenced, f"MEMBAR.ALL.GPU in the slot release after a wgmma wait (kernel: windows): {fenced}"
