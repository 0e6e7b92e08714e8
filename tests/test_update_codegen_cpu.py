"""What the compiler makes of the fused weight-update kernels (optim_tc.cu), checked without a GPU.

The update moves about 0.75 GB per Large train step and is bound by how many bytes each SM keeps in flight.  The source
is compiled for sm_90a with the library's own flags, and for every instantiation of update_pack_kernel and
update_pack_whh_kernel (4 / 2 / 1 columns per thread x SgdRule / DynRule<false> / DynRule<true>) three properties
the speed rests on are held:

- no CALL: the tile index arithmetic is 32-bit, so no 64-bit division subroutine is called.  The one exception is
  DynRule<true>, whose element rule (dyneval_elem) divides by r + eps with a correctly rounded fp32 division; its only
  calls go to that division's slow path.
- a 0-byte stack frame: the tile of 8 rows x 4 columns of g and p (and theta_g, r) stays in registers.  The kernels
  before the tiles had one too; this guards against spills of the larger per-thread tile (DynRule<true> calls the
  division slow path, and values kept live across those calls have spilled).
- every global load of the tile is issued before the first global store: the thread's loads are all in flight at once
  instead of one dependent DRAM round trip per row.

Skipped without nvcc, like the other host-compiled checks.
"""
import os
import re
import shutil
import subprocess

import pytest

from zaremba_b200 import build as zb

SOURCE = os.path.join(zb.CSRC, "optim_tc.cu")
RULES = {"SgdRule": "NS_7SgdRule", "DynRule<false>": "NS_7DynRuleILb0E", "DynRule<true>": "NS_7DynRuleILb1E"}
INSTANCES = [(k, v, r) for k in ("update_pack_kernel", "update_pack_whh_kernel") for v in (4, 2, 1) for r in RULES]


def _tool(name):
    for c in (shutil.which(name), f"/usr/local/cuda/bin/{name}"):
        if c and os.path.exists(c):
            return c
    pytest.skip(f"{name} is not available")


@pytest.fixture(scope="module")
def codegen(tmp_path_factory):
    """(ptxas -v log, {mangled kernel name: [SASS instruction lines]})"""
    try:
        nvcc = zb._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not available")
    flags = [f for f in zb.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cubin = str(tmp_path_factory.mktemp("update_codegen") / "optim_tc.cubin")
    r = subprocess.run([nvcc, *flags, "-Xptxas", "-v", "--cubin", SOURCE, "-o", cubin],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout
    dis = subprocess.run([_tool("nvdisasm"), cubin], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         timeout=600)
    assert dis.returncode == 0, dis.stdout
    kernels, cur = {}, None
    for line in dis.stdout.splitlines():
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", line)
        if m:
            cur = kernels.setdefault(m.group(1), [])
            continue
        if re.match(r"\s*\.section", line):
            cur = None
        elif cur is not None and re.search(r"/\*[0-9a-f]{4,}\*/", line):
            cur.append(line)
    return r.stdout, kernels


def _mangled(kernel, vec, rule, names):
    found = [n for n in names if f"{len(kernel)}{kernel}ILi{vec}E{RULES[rule]}" in n]
    assert len(found) == 1, (kernel, vec, rule, found)
    return found[0]


def _ids():
    return [f"{k}<{v},{r}>" for k, v, r in INSTANCES]


def test_every_instantiation_is_compiled(codegen):
    _, kernels = codegen
    names = [n for n in kernels if "update_pack" in n]
    assert len(names) == len(INSTANCES), names
    for k, v, r in INSTANCES:
        _mangled(k, v, r, names)


@pytest.mark.parametrize("kernel,vec,rule", INSTANCES, ids=_ids())
def test_no_call(kernel, vec, rule, codegen):
    _, kernels = codegen
    sass = kernels[_mangled(kernel, vec, rule, kernels)]
    calls = [line.strip() for line in sass if re.search(r"\bCALL\b", line)]
    if rule == "DynRule<true>":
        calls = [c for c in calls if "div_rn_noftz_f32_slowpath" not in c]
    assert not calls, calls
    assert not any(re.search(r"_(div|rem)_[su](32|64)", line) for line in sass)


@pytest.mark.parametrize("kernel,vec,rule", INSTANCES, ids=_ids())
def test_zero_stack_frame(kernel, vec, rule, codegen):
    log, kernels = codegen
    name = _mangled(kernel, vec, rule, kernels)
    m = re.search(r"Function properties for " + re.escape(name) + r"\s*\n\s*(\d+) bytes stack frame", log)
    assert m, log
    assert int(m.group(1)) == 0


@pytest.mark.parametrize("kernel,vec,rule", INSTANCES, ids=_ids())
def test_every_load_is_issued_before_the_first_store(kernel, vec, rule, codegen):
    _, kernels = codegen
    sass = kernels[_mangled(kernel, vec, rule, kernels)]
    loads = [i for i, line in enumerate(sass) if re.search(r"\bLDG\b|\bLDG\.", line)]
    stores = [i for i, line in enumerate(sass) if re.search(r"\bSTG\b|\bSTG\.", line)]
    assert loads and stores
    assert max(loads) < min(stores), (sass[min(stores)].strip(), sass[max(loads)].strip())
