"""Iterate averaging (NT-ASGD, DESIGN.md section 16) without a GPU.

- The numpy restatement (tests/_asgd_oracle.py) against torch.optim.ASGD(lambd=0, t0=0), bit for bit.  torch's mu runs
  one step behind its step counter (its first two updates both copy), so after k torch steps its average equals the
  restatement started at torch step 2, i.e. over the last k - 1 weight vectors.
- The C ABI: header prototypes, ctypes bindings, refusals that need no context.
- What the compiler makes of the averaged tile kernels and the swap kernels (average_tc.cu), as
  tests/test_update_codegen_cpu.py holds it for optim_tc.cu: no CALL, a 0-byte stack frame, and every global load of
  a tile issued before its first store; a 0-byte stack frame for the list kernels.  Skipped without nvcc.
"""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests import _asgd_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the restatement ------------------------------------------------------------------------------------------------
def test_mu_is_rounded_once_from_double():
    for n in (1, 2, 3, 7, 10, 1000, 3 * 2 ** 20 + 1):
        assert AO.mu(n) == np.float32(1.0 / n)


def test_first_update_copies_even_garbage():
    a = np.array([np.nan, np.inf, -1e30], dtype=np.float32)
    th = np.array([1.0, 2.0, 3.0], dtype=np.float32)
    out = AO.avg_update(a, th, 1)
    assert out.tobytes() == th.tobytes()


def test_restart_keeps_contents_and_resets_n():
    av = AO.Averager()
    rng = np.random.default_rng(0)
    for _ in range(3):
        av.update(rng.standard_normal(8).astype(np.float32))
    kept = av.a.copy()
    av.start()
    assert av.n == 0 and av.a.tobytes() == kept.tobytes()
    th = rng.standard_normal(8).astype(np.float32)
    assert av.update(th).tobytes() == th.tobytes() and av.n == 1


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_equals_torch_asgd(seed):
    """theta / gradient sequence through torch.optim.ASGD(lambd=0, t0=0, weight_decay=0); the restatement, fed torch's
    own theta after every step from step 2 on, reproduces torch's ax bit for bit at every step."""
    g = torch.Generator().manual_seed(seed)
    p = torch.nn.Parameter(torch.randn(1000, generator=g))
    opt = torch.optim.ASGD([p], lr=0.5, lambd=0.0, alpha=0.75, t0=0.0, weight_decay=0.0, foreach=False)
    av = AO.Averager()
    for k in range(1, 40):
        p.grad = torch.randn(1000, generator=g) * (1.0 + k)
        opt.step()
        theta = p.detach().numpy()
        ax = opt.state[p]["ax"].numpy()
        if k == 1:
            assert ax.tobytes() == theta.tobytes()
            continue
        a = av.update(theta)
        assert av.n == k - 1
        assert a.tobytes() == ax.tobytes(), f"step {k}: max |diff| {np.abs(a - ax).max()}"


def test_restatement_is_the_running_mean():
    rng = np.random.default_rng(5)
    thetas = [rng.standard_normal(64) for _ in range(50)]
    av = AO.Averager()
    for th in thetas:
        av.update(np.float32(th))
    np.testing.assert_allclose(av.a, np.mean(np.float32(thetas), axis=0), rtol=0, atol=1e-5)


# ---- C ABI ----------------------------------------------------------------------------------------------------------
PROTOS = {
    "zrb_set_average": r"int\s+zrb_set_average\(zrb_ctx\* ctx, const zrb_params\* avg\);",
    "zrb_average_count": r"int\s+zrb_average_count\(const zrb_ctx\* ctx, int64_t\* n\);",
    "zrb_swap_average": r"int\s+zrb_swap_average\(zrb_ctx\* ctx, const zrb_params\* p, void\* stream\);",
}


def test_header_and_bindings():
    from zaremba_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "zaremba_b200.h")).read()
    for name, proto in PROTOS.items():
        assert re.search(proto, hdr), name
        assert name in _lib.exported_symbols(), name
    P = C.POINTER(_lib.ZrbParams)
    assert _lib._SIGNATURES["zrb_set_average"] == (C.c_int, [C.c_void_p, P])
    assert _lib._SIGNATURES["zrb_average_count"] == (C.c_int, [C.c_void_p, C.POINTER(C.c_int64)])
    assert _lib._SIGNATURES["zrb_swap_average"] == (C.c_int, [C.c_void_p, P, C.c_void_p])
    import zaremba_b200
    for m in ("start_averaging", "stop_averaging", "averaged_weights", "average_state_dict"):
        assert callable(getattr(zaremba_b200.Trainer, m)), m
    assert isinstance(zaremba_b200.Trainer.averaged_steps, property)


def test_null_context_is_refused():
    from zaremba_b200 import _lib
    try:
        lib = _lib.load()
    except Exception as e:   # no library and no nvcc: nothing to call
        pytest.skip(f"library unavailable: {e}")
    ps = _lib.ZrbParams()
    n = C.c_int64(7)
    assert lib.zrb_set_average(None, C.byref(ps)) == -1
    assert lib.zrb_set_average(None, None) == -1
    assert lib.zrb_average_count(None, C.byref(n)) == -1 and n.value == 7
    assert lib.zrb_swap_average(None, C.byref(ps), None) == -1


# ---- codegen of average_tc.cu ----------------------------------------------------------------------------------------
RULES = {"AvgRule": "NS_7AvgRuleE", "SwapRule": "NS_8SwapRuleE"}
INSTANCES = [(k, v, r) for k in ("update_pack_kernel", "update_pack_whh_kernel") for v in (4, 2, 1) for r in RULES]
LIST_KERNELS = ["sgd_avg_list_kernelILb1ELb1E", "sgd_avg_list_kernelILb1ELb0E", "sgd_avg_list_kernelILb0ELb0E",
                "swap_list_kernel"]


def _tool(name):
    for c in (shutil.which(name), f"/usr/local/cuda/bin/{name}"):
        if c and os.path.exists(c):
            return c
    pytest.skip(f"{name} is not available")


@pytest.fixture(scope="module")
def codegen(tmp_path_factory):
    """(ptxas -v log, {mangled kernel name: [SASS instruction lines]}) of average_tc.cu"""
    from zaremba_b200 import build as zb
    try:
        nvcc = zb._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not available")
    flags = [f for f in zb.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cubin = str(tmp_path_factory.mktemp("average_codegen") / "average_tc.cubin")
    r = subprocess.run([nvcc, *flags, "-Xptxas", "-v", "--cubin", os.path.join(zb.CSRC, "average_tc.cu"), "-o", cubin],
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


def _tile_pattern(kernel, vec, rule):
    return f"{len(kernel)}{kernel}ILi{vec}E{RULES[rule]}"


def _ids():
    return [f"{k}<{v},{r}>" for k, v, r in INSTANCES]


def test_every_instantiation_is_compiled(codegen):
    _, kernels = codegen
    assert len([n for n in kernels if "update_pack" in n]) == len(INSTANCES), sorted(kernels)
    for k, v, r in INSTANCES:
        _mangled(_tile_pattern(k, v, r), kernels)
    for k in LIST_KERNELS:
        _mangled(k, kernels)


def _all_names():
    return [_tile_pattern(k, v, r) for k, v, r in INSTANCES] + LIST_KERNELS


@pytest.mark.parametrize("kernel,vec,rule", INSTANCES, ids=_ids())
def test_no_call(kernel, vec, rule, codegen):
    """The tile kernels' index arithmetic is 32-bit.  (The list kernels' grid-stride loops divide in 64 bits once per
    thread, as sgd_apply's do.)"""
    _, kernels = codegen
    sass = kernels[_mangled(_tile_pattern(kernel, vec, rule), kernels)]
    assert not [line for line in sass if re.search(r"\bCALL\b", line)]
    assert not any(re.search(r"_(div|rem)_[su](32|64)", line) for line in sass)


@pytest.mark.parametrize("pattern", _all_names())
def test_zero_stack_frame(pattern, codegen):
    log, kernels = codegen
    name = _mangled(pattern, kernels)
    m = re.search(r"Function properties for " + re.escape(name) + r"\s*\n\s*(\d+) bytes stack frame", log)
    assert m, log
    assert int(m.group(1)) == 0


@pytest.mark.parametrize("kernel,vec,rule", INSTANCES, ids=_ids())
def test_every_load_is_issued_before_the_first_store(kernel, vec, rule, codegen):
    _, kernels = codegen
    sass = kernels[_mangled(_tile_pattern(kernel, vec, rule), kernels)]
    loads = [i for i, line in enumerate(sass) if re.search(r"\bLDG\b|\bLDG\.", line)]
    stores = [i for i, line in enumerate(sass) if re.search(r"\bSTG\b|\bSTG\.", line)]
    assert loads and stores
    assert max(loads) < min(stores), (sass[min(stores)].strip(), sass[max(loads)].strip())
