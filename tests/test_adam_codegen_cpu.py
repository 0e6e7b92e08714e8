"""What the compiler makes of the Adam update kernels (adam_tc.cu), checked without a GPU, as
tests/test_update_codegen_cpu.py holds it for optim_tc.cu.  For every instantiation of update_pack_kernel and
update_pack_whh_kernel with AdamRule (4 / 2 / 1 columns per thread):

- no CALL but the slow paths of the correctly rounded fp32 division and square root, and no 64-bit integer division;
- a 0-byte stack frame: the tiles of g, p, m and v (128 values at 4 columns) stay in registers, also across those calls;
- every global load of the tile is issued before the first global store.

The list kernels get the 0-byte stack frame check.  Skipped without nvcc.
"""
import os
import re
import shutil
import subprocess

import pytest

from zaremba_b200 import build as zb

SOURCE = os.path.join(zb.CSRC, "adam_tc.cu")
INSTANCES = [(k, v) for k in ("update_pack_kernel", "update_pack_whh_kernel") for v in (4, 2, 1)]
LIST_KERNELS = ["adam_list_kernelILb1E", "adam_list_kernelILb0E"]
SLOW_PATHS = ("div_rn_noftz_f32_slowpath", "sqrt_rn_f32_slowpath")


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
    cubin = str(tmp_path_factory.mktemp("adam_codegen") / "adam_tc.cubin")
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


def _mangled(pattern, names):
    found = [n for n in names if pattern in n]
    assert len(found) == 1, (pattern, found)
    return found[0]


def _tile_pattern(kernel, vec):
    return f"{len(kernel)}{kernel}ILi{vec}ENS_8AdamRuleE"


def _ids():
    return [f"{k}<{v},AdamRule>" for k, v in INSTANCES]


def test_every_instantiation_is_compiled(codegen):
    _, kernels = codegen
    assert len([n for n in kernels if "update_pack" in n]) == len(INSTANCES), sorted(kernels)
    for k, v in INSTANCES:
        _mangled(_tile_pattern(k, v), kernels)
    for k in LIST_KERNELS:
        _mangled(k, kernels)


@pytest.mark.parametrize("kernel,vec", INSTANCES, ids=_ids())
def test_no_call(kernel, vec, codegen):
    _, kernels = codegen
    sass = kernels[_mangled(_tile_pattern(kernel, vec), kernels)]
    calls = [line.strip() for line in sass if re.search(r"\bCALL\b", line)]
    assert not [c for c in calls if not any(s in c for s in SLOW_PATHS)], calls
    assert not any(re.search(r"_(div|rem)_[su](32|64)", line) for line in sass)


@pytest.mark.parametrize("pattern", [_tile_pattern(k, v) for k, v in INSTANCES] + LIST_KERNELS)
def test_zero_stack_frame(pattern, codegen):
    log, kernels = codegen
    name = _mangled(pattern, kernels)
    m = re.search(r"Function properties for " + re.escape(name) + r"\s*\n\s*(\d+) bytes stack frame", log)
    assert m, log
    assert int(m.group(1)) == 0


@pytest.mark.parametrize("kernel,vec", INSTANCES, ids=_ids())
def test_every_load_is_issued_before_the_first_store(kernel, vec, codegen):
    _, kernels = codegen
    sass = kernels[_mangled(_tile_pattern(kernel, vec), kernels)]
    loads = [i for i, line in enumerate(sass) if re.search(r"\bLDG\b|\bLDG\.", line)]
    stores = [i for i, line in enumerate(sass) if re.search(r"\bSTG\b|\bSTG\.", line)]
    assert loads and stores
    assert max(loads) < min(stores), (sass[min(stores)].strip(), sass[max(loads)].strip())
