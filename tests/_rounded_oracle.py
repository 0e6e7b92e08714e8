"""One LSTM layer restated on the operands the tensor-core kernels multiply  --  TEST INFRASTRUCTURE
(tests/_trained_regime.py, tests/test_gpu_rec_bwd_images.py, tests/test_rounded_oracle_cpu.py).

Forward and backward in fp64 (torch, on any device), each step teacher-forced on what the device produced: the forward
on the device's fp16 image of h_{t-1}, the backward on the device's fp16 image of dG_{t+1} (kGradScale * dG, clamped to
+-65504).  A rounding flip in one image then cannot propagate, and what remains between a kernel and this restatement
is one step of fp32 arithmetic and the activation functions: small enough to hold element by element.

Every quantity carries a magnitude E >= |value| (the class `M`): sums add magnitudes, a product a * b has
E(a) |b| + |a| E(b), and an activation output v = act(z) has |v| + 1 + |act'(z)| E(z) -- the 1 because the SFU and libm
activations are accurate to a few fp32 ulp absolutely, not relatively, which is what matters where 1 - g cancels at a
saturated gate.  An fp32 evaluation of the same expression differs from the fp64 value by a small multiple of
2^-24 * E, element by element; the tests hold that multiple (tau) to what they measure.
"""
from __future__ import annotations

import numpy as np
import torch

GRAD_SCALE = 1024.0          # tc_kernels.h kGradScale
F16_MAX = 65504.0
F16_MIN_NORMAL = 2.0 ** -14


def r16(a):
    """fp16 rounding (round to nearest even), in fp64."""
    return a.to(torch.float16).to(torch.float64)


def ulp16(v):
    """The spacing of fp16 values at |v| (v fp16-representable): 2^-24 below the normal range."""
    e = torch.floor(torch.log2(v.abs().clamp(min=F16_MIN_NORMAL)))
    return torch.exp2(e - 10.0)


def image(dG):
    """The fp16 image the kernels store for a gate gradient: fp16(clamp(kGradScale * dG, +-65504))."""
    return r16((GRAD_SCALE * dG).clamp(-F16_MAX, F16_MAX))


def rescale_image(y, k):
    """The image r(k h) of a value h known only through its image y = r(h) (k = 2) or y = r(2 h) (k = 1/2): (best
    value, absolute uncertainty).  Doubling or halving a normal fp16 value is exact; below the normal range the
    quantum stays 2^-24, so one bit of the other image is unknown (halving: only where y / 2^-24 is odd)."""
    if k == 2:
        return 2.0 * y, torch.where(y.abs() <= F16_MIN_NORMAL, 2.0 ** -24, 0.0).to(y)
    assert k == 0.5
    odd = (y.abs() < 2.0 * F16_MIN_NORMAL) & (torch.remainder(y * 2.0 ** 24, 2.0) == 1.0)
    return 0.5 * y, torch.where(odd, 2.0 ** -25, 0.0).to(y)


class M:
    """A value and its magnitude E (see the module docstring)."""

    def __init__(self, v, e=None):
        self.v = v
        self.e = v.abs() if e is None else e

    def __getitem__(self, k):
        return M(self.v[k], self.e[k])

    def __add__(self, o):
        o = _m(o, self.v)
        return M(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = _m(o, self.v)
        return M(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return _m(o, self.v) - self

    def __mul__(self, o):
        o = _m(o, self.v)
        return M(self.v * o.v, self.e * o.v.abs() + self.v.abs() * o.e)

    __rmul__ = __mul__


def _m(o, like):
    return o if isinstance(o, M) else M(torch.full_like(like, float(o)))


def sigmoid(z):
    v = torch.sigmoid(z.v)
    return M(v, v.abs() + 1.0 + v * (1.0 - v) * z.e)


def tanh(z):
    v = torch.tanh(z.v)
    return M(v, v.abs() + 1.0 + (1.0 - v * v) * z.e)


def where(cond, a, b):
    return M(torch.where(cond, a.v, b.v), torch.where(cond, a.e, b.e))


def matmul(a, W):
    """a @ W for an exact operand a: E = |a| @ |W|."""
    return M(a @ W, a.abs() @ W.abs())


def forward(pre, Wr, c0, a=None, h0=None, q=None, zc=None, zh=None, rnd=r16):
    """Forward of one layer.  pre [T,B,4H]: the input GEMM's result (M, fp64); Wr [4H,H]: the W_hh the kernels hold;
    a [T,B,H]: the recurrent operand of each step, the device's image of q * h_{t-1} (teacher-forced) -- None: the
    restatement's own, rnd(q * h_{t-1}) with h_{-1} = h0; q [B,H]: the variational mode's recurrent multiplier (None: 1);
    zc, zh [T,B,H] bool: zoneout flags, True = the unit keeps its previous c / h.
    Returns {"z", "i", "f", "g", "o", "c" (after zoneout), "ct" (c~), "h" (after zoneout, own path), "hn" (the new h~)}:
    lists over t of M."""
    T = pre.v.shape[0]
    c = M(c0)
    h = h0
    out = {k: [] for k in ("z", "i", "f", "g", "o", "c", "ct", "h", "hn")}
    for t in range(T):
        if a is not None:
            at = a[t]
        else:
            at = rnd(h if q is None else q * h)
        z = pre[t] + matmul(at, Wr.T)
        H = Wr.shape[1]
        zi, zf, zg, zo = (M(z.v[:, k * H:(k + 1) * H], z.e[:, k * H:(k + 1) * H]) for k in range(4))
        i, f, g, o = sigmoid(zi), sigmoid(zf), tanh(zg), sigmoid(zo)
        ct = f * c + i * g
        hn = o * tanh(ct)
        cn = ct if zc is None else where(zc[t], c, ct)
        if a is None:
            h = hn.v if zh is None else torch.where(zh[t], h, hn.v)
        for k, v in (("z", z), ("i", i), ("f", f), ("g", g), ("o", o), ("c", cn), ("ct", ct), ("hn", hn)):
            out[k].append(v)
        out["h"].append(h)
        c = cn
    return out


MUTATIONS = ("drop_partial", "stale_slot", "flush_subnormal", "shift_column", "multiplier_on_dy", "drop_hcarry")


def backward(fw, dyv, Wr, c0, img=None, q=None, zc=None, zh=None, rounded=True, mutate=None, geometry=None):
    """Backward of one layer along the forward `fw` (forward's dict).  dyv [T,B,H]: the upstream gradient after the
    output dropout (exact); img [T,B,4H]: the device's dG images, step t uses img[t+1] (teacher-forced) -- None: the
    restatement's own image of dG_{t+1} (rounded=True) or exact 1024 dG_{t+1} (rounded=False).  dc and the zoneout
    h-carry are carried in fp64.  Returns (dG [T,B,4H] value, E).
    mutate: one of MUTATIONS, a deliberate error of the kernel's kind, so that a test can show its bound resolves it;
    geometry = (rows, units) for "drop_partial": the W_hh rows one cluster CTA contracts and the units it sends them to."""
    T, B, H = dyv.shape
    dG, dGe = torch.zeros(T, B, 4 * H).to(dyv), torch.zeros(T, B, 4 * H).to(dyv)
    dc = M(torch.zeros(B, H).to(dyv))
    hcarry = M(torch.zeros(B, H).to(dyv))
    own = None
    for t in range(T - 1, -1, -1):
        dh = M(dyv[t])
        if t < T - 1:
            nxt = own if img is None else img[t + 1]
            if mutate == "stale_slot":
                nxt = img[t]
            elif mutate == "flush_subnormal":
                nxt = torch.where(nxt.abs() < F16_MIN_NORMAL, 0.0, nxt)
            elif mutate == "shift_column":
                g0 = 8 * ((B - 1) // 8)
                nxt = torch.cat([nxt[:g0], nxt[g0 + 1:], torch.zeros_like(nxt[:1])])
            rec = matmul(nxt, Wr)
            if mutate == "drop_partial":
                rows, units = geometry
                rec.v[:, units] -= nxt[:, rows] @ Wr[rows][:, units]
            rec = M(rec.v / GRAD_SCALE, rec.e / GRAD_SCALE)
            if q is not None and mutate == "multiplier_on_dy":
                dh = M(dyv[t] * q) + rec
            else:
                dh = dh + (rec if q is None else rec * M(q))
        if zh is not None:
            if mutate != "drop_hcarry":
                dh = dh + hcarry
            zero = M(torch.zeros_like(dh.v))
            hcarry = where(zh[t], dh, zero)
            dh = where(zh[t], zero, dh)
        i, f, g, o = fw["i"][t], fw["f"][t], fw["g"][t], fw["o"][t]
        tc = tanh(fw["ct"][t])
        c_prev = fw["c"][t - 1] if t > 0 else M(c0)
        dt = dh * o * (1.0 - tc * tc)
        dcc = dc + dt if zc is None else where(zc[t], dt, dc + dt)
        d_i, d_f, d_g, d_o = dcc * g, dcc * c_prev, dcc * i, dh * tc
        dc = dcc * f if zc is None else where(zc[t], dcc * f + dc, dcc * f)
        gates = [d_i * (i * (1.0 - i)), d_f * (f * (1.0 - f)), d_g * (1.0 - g * g), d_o * (o * (1.0 - o))]
        dG[t] = torch.cat([x.v for x in gates], 1)
        dGe[t] = torch.cat([x.e for x in gates], 1)
        own = image(dG[t]) if rounded else GRAD_SCALE * dG[t]
    return dG, dGe


def rounded_operand_fwd(x, h0, c0, W_ih, W_hh, b_ih, b_hh, h_dev):
    """fp64 forward of one layer fed exactly what the tensor-core kernels multiply -- fp16-rounded x, W_ih, W_hh and
    h_{t-1} -- with exact activations.  h_{t-1} is the DEVICE's h (h_dev [T,B,H]; h0 at t = 0), so that a rounding flip
    of one fp16 h image cannot propagate: what remains between the device and this is fp32 accumulation and the
    activation functions.  numpy in and out.  Returns y [T,B,H], c_T and the largest |pre-activation|."""
    f = lambda v: torch.as_tensor(np.asarray(v, dtype=np.float64))
    x, h0, h_dev = f(x), f(h0), f(h_dev)
    pre = M(r16(x) @ r16(f(W_ih)).T + f(b_ih) + f(b_hh))
    a = r16(torch.cat([h0[None], h_dev[:-1]]))
    fw = forward(pre, r16(f(W_hh)), f(c0), a=a)
    return (torch.stack([h.v for h in fw["hn"]]).numpy(), fw["c"][-1].v.numpy(),
            float(max(z.v.abs().max() for z in fw["z"])))


def layer(x, h0, c0, W_ih, W_hh, b_ih, b_hh, dy, rounded=True):
    """Forward and backward of one layer, each step forced on the restatement's own images: with rounded=True the
    images the kernels would hold (fp16 operands, fp16 dG images), with rounded=False exact values -- then this is
    oracle.lstm_layer_fwd / lstm_layer_bwd.  torch fp64 in.  Returns (fw, dG, E, dx, dW_ih, dW_hh, db)."""
    rnd = r16 if rounded else (lambda v: v)
    T, B, _ = x.shape
    xr, Wr = rnd(x), rnd(W_hh)
    pre = M(xr @ rnd(W_ih).T + b_ih + b_hh)
    fw = forward(pre, Wr, c0, h0=h0, rnd=rnd)
    dG, E = backward(fw, dy, Wr, c0, rounded=rounded)
    hprev = rnd(torch.stack([h0] + fw["h"][:-1]))
    N = T * B
    return (fw, dG, E, dG @ W_ih, dG.reshape(N, -1).T @ xr.reshape(N, -1), dG.reshape(N, -1).T @ hprev.reshape(N, -1),
            dG.sum((0, 1)))
