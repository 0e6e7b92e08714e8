"""What ptxas makes of the library's wgmma code, checked without a GPU.

Every CUDA source is compiled for sm_90a with the library's own flags plus `-Xptxas -v`, and two properties that
tests on a GPU would only see as a slower step are held:

- no wgmma chain is serialised.  ptxas reports C7520 ("wgmma.mma_async instructions are serialized") when a call or a
  branch it cannot prove warp-uniform sits between wgmmas whose accumulators are live; it then waits for each wgmma
  before issuing the next, and a chain of 94 wgmmas pays 94 full latencies per recurrence step.
- the persistent recurrence kernels keep nothing in local memory (0-byte stack frame, so no register spills either):
  their per-step loops would otherwise reload kernel arguments and flags from it every step.

Skipped without nvcc, like the other host-compiled checks.
"""
import os
import re
import subprocess

import pytest

from zaremba_b200 import build as zb

SOURCES = [os.path.basename(s) for s in zb.sources()]
REC_KERNELS = {"lstm_rec_fwd.cu": 2, "lstm_rec_bwd.cu": 2}   # instantiations of the persistent kernel in each source


@pytest.fixture(scope="module")
def ptxas_logs(tmp_path_factory):
    """{source: ptxas -v output}, every source compiled as the library compiles it (device code only), all at once."""
    try:
        nvcc = zb._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not available")
    flags = [f for f in zb.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    out = tmp_path_factory.mktemp("codegen")
    procs = {name: subprocess.Popen([nvcc, *flags, "-Xptxas", "-v", "--cubin", os.path.join(zb.CSRC, name),
                                     "-o", str(out / (name[:-3] + ".cubin"))],
                                    stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for name in SOURCES}
    logs = {}
    for name, p in procs.items():
        logs[name] = p.communicate(timeout=1800)[0]
        assert p.returncode == 0, logs[name]
    return logs


def _stack_frames(log):
    """{mangled function name: stack frame bytes} from ptxas -v."""
    return {m.group(1): int(m.group(2))
            for m in re.finditer(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame", log)}


def test_the_recurrence_and_gemm_sources_are_covered():
    assert set(REC_KERNELS) <= set(SOURCES) and "gemm_tc.cu" in SOURCES


@pytest.mark.parametrize("name", SOURCES)
def test_no_serialized_wgmma(name, ptxas_logs):
    bad = [line for line in ptxas_logs[name].splitlines()
           if "C7520" in line or "wgmma.mma_async instructions are serialized" in line]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("name", sorted(REC_KERNELS))
def test_recurrence_kernels_use_no_local_memory(name, ptxas_logs):
    frames = _stack_frames(ptxas_logs[name])
    kernels = {f: b for f, b in frames.items() if re.search(r"lstm_rec_(fwd|bwd)_kernel", f)}
    assert len(kernels) == REC_KERNELS[name], frames
    assert all(b == 0 for b in kernels.values()), kernels
