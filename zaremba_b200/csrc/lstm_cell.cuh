// The LSTM cell's pointwise rule (model.py:37-45, nn.LSTM's (i,f,g,o) order; zoneout: DESIGN.md section 20), written
// once for every kernel that runs it: the validation engine's (pointwise.cu), the tensor-core engine's per-timestep
// kernels (tc_cell.cu) and the persistent recurrences (lstm_rec_fwd.cuh, lstm_rec_bwd.cuh).  The kernels keep their own
// loads, stores, masks and operand images; these functions are the arithmetic between them.
#pragma once
#include "tc_kernels.h"

namespace zrb {

// Activation policies.  The validation engine and the per-timestep kernels take PreciseAct, the persistent kernels
// FastAct: sigmoid / tanh on the SFU exp path (abs error ~1e-7, far below the fp16 operand noise of that engine).
struct PreciseAct {
    __device__ static float sigmoid(float z) { return 1.f / (1.f + expf(-z)); }
    __device__ static float tanh(float x) { return tanhf(x); }
};
struct FastAct {
    __device__ __forceinline__ static float sigmoid(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
    __device__ __forceinline__ static float tanh(float x) { return 1.f - __fdividef(2.f, 1.f + __expf(2.f * x)); }
};

struct CellFwd {
    float i, f, g, o;   // the activated gates
    float ctil;         // c~ = fma(i, g, f c_prev) (the backward's c_t under zoneout)
    float c, h;         // the carried state: c~ and h~ = o tanh(c~), or their zoned values
};

// Forward of one cell from its four pre-activations.  ZO, train mode (zo.flags set): the cell keeps c_prev where kc is set
// and h_prev where kh is (a select, no scaling, no rounding); eval mode (zo.flags null): the expectation
// fma(z, prev, (1 - z) new).
template <class Act, bool ZO>
__device__ __forceinline__ CellFwd cell_fwd(float zi, float zf, float zg, float zo_, float c_prev, float h_prev,
                                            bool kc, bool kh, const ZoneoutSrc& zo) {
    const float i = Act::sigmoid(zi), f = Act::sigmoid(zf), g = Act::tanh(zg), o = Act::sigmoid(zo_);
    const float ctil = __fmaf_rn(i, g, __fmul_rn(f, c_prev));   // (spelled out: the compiler may contract it either way)
    float c = ctil, h = o * Act::tanh(ctil);
    if constexpr (ZO) {
        if (zo.flags) {
            if (kc) c = c_prev;
            if (kh) h = h_prev;
        } else {
            c = __fmaf_rn(zo.ec, c_prev, __fmul_rn(zo.ec1, c));
            h = __fmaf_rn(zo.eh, h_prev, __fmul_rn(zo.eh1, h));
        }
    }
    return {i, f, g, o, ctil, c, h};
}

struct CellGrad { float i, f, g, o; };   // dG: the gradients of the four pre-activations

// Backward of one cell from its saved gates, c_t (ZO: c~_t) and c_prev.  dh is the whole gradient of h_t, assembled by the
// caller (the kernels add its terms in different orders); dc carries dc_t in and dc_{t-1} out.  ZO (kc, kh and zo as
// in cell_fwd): dh~ = (1 - zh) dh, dc~ = (1 - zc) dc + dh~ o (1 - tanh^2 c~), dc_{t-1} = zc dc + f dc~, and hcarry receives
// zh dh, which the caller adds to dh_{t-1}.
template <class Act, bool ZO>
__device__ __forceinline__ CellGrad cell_bwd(float i, float f, float g, float o, float c_t, float c_prev, float dh,
                                             float& dc, float& hcarry, bool kc, bool kh, const ZoneoutSrc& zo) {
    if constexpr (ZO) {
        const float dht = zo.flags ? (kh ? 0.f : dh) : __fmul_rn(zo.eh1, dh);
        hcarry = zo.flags ? (kh ? dh : 0.f) : __fmul_rn(zo.eh, dh);
        dh = dht;
    }
    const float tc = Act::tanh(c_t);
    const float d_o = dh * tc;
    float dcc;
    if constexpr (ZO) {   // dc~: the carried dc times (1 - zc), plus the h~ path (h~ reads c~)
        const float dt = __fmul_rn(__fmul_rn(dh, o), __fsub_rn(1.f, __fmul_rn(tc, tc)));
        dcc = zo.flags ? (kc ? dt : __fadd_rn(dc, dt)) : __fmaf_rn(zo.ec1, dc, dt);
    } else {
        dcc = dc + dh * o * (1.f - tc * tc);
    }
    const float d_i = dcc * g, d_g = dcc * i, d_f = dcc * c_prev;
    if constexpr (ZO)
        dc = zo.flags ? (kc ? __fmaf_rn(dcc, f, dc) : __fmul_rn(dcc, f)) : __fmaf_rn(zo.ec, dc, __fmul_rn(dcc, f));
    else
        dc = dcc * f;
    return {d_i * i * (1.f - i), d_f * f * (1.f - f), d_g * (1.f - g * g), d_o * o * (1.f - o)};
}

}  // namespace zrb
