// Pointwise kernels of the tensor-core engine: same math as pointwise.cu, plus the fp16 operand
// images the tensor-core GEMMs consume (h_t for the next step / wgrad, dropout(h_t) for the next
// layer, scaled dG and dS).  HBM/L2-bound, fully coalesced.
#include "tc_kernels.h"

namespace zrb {

__global__ void lstm_cell_fwd_tc_kernel(float* __restrict__ pre, const float* __restrict__ c_prev,
                                        float* __restrict__ c_out, float* __restrict__ h_raw,
                                        __half* __restrict__ h_raw_h, __half* __restrict__ y_h, int64_t ld_h, int B,
                                        int H, int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (int64_t)B * H) return;
    int b = (int)(tid / H), j = (int)(tid % H);
    float* row = pre + (int64_t)b * 4 * H;
    float i = sigmoidf_(row[j]);
    float f = sigmoidf_(row[H + j]);
    float g = tanhf(row[2 * H + j]);
    float o = sigmoidf_(row[3 * H + j]);
    float c = f * c_prev[tid] + i * g;
    float h = o * tanhf(c);
    row[j] = i; row[H + j] = f; row[2 * H + j] = g; row[3 * H + j] = o;
    c_out[tid] = c;
    h_raw[tid] = h;
    h_raw_h[(int64_t)b * ld_h + j] = __float2half_rn(h * mask_mul1_at(rm, (uint64_t)tid, (uint64_t)B * H));   // next step's operand
    y_h[(int64_t)b * ld_h + j] = __float2half_rn(h * mask_mul1(m, (uint64_t)(elem_off + tid), (uint64_t)n_total));
}

int lstm_cell_fwd_tc(float* pre, const float* c_prev, float* c_out, float* h_raw, __half* h_raw_h, __half* y_h,
                     int64_t ld_h, int B, int H, int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s) {
    int64_t n = (int64_t)B * H;
    lstm_cell_fwd_tc_kernel<<<cdiv(n, 256), 256, 0, s>>>(pre, c_prev, c_out, h_raw, h_raw_h, y_h, ld_h, B, H, elem_off,
                                                         n_total, m, rm);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

__device__ __forceinline__ __half to_half_scaled(float v) {
    v *= kGradScale;
    v = fminf(fmaxf(v, -65504.f), 65504.f);
    return __float2half_rn(v);
}

__global__ void lstm_cell_bwd_tc_kernel(const float* __restrict__ dy_post, const float* __restrict__ dh_rec,
                                        float* __restrict__ dc, const float* __restrict__ gates,
                                        const float* __restrict__ c_t, const float* __restrict__ c_prev,
                                        float* __restrict__ dG, __half* __restrict__ dG_h, int64_t ld_g, int B, int H,
                                        int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm,
                                        const float* __restrict__ r) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (int64_t)B * H) return;
    int b = (int)(tid / H), j = (int)(tid % H);
    const float* row = gates + (int64_t)b * 4 * H;
    float i = row[j], f = row[H + j], g = row[2 * H + j], o = row[3 * H + j];
    float dh = dy_post[tid] * mask_mul1(m, (uint64_t)(elem_off + tid), (uint64_t)n_total);
    if (r) dh += r[tid];
    if (dh_rec) dh += dh_rec[tid] * mask_mul1_at(rm, (uint64_t)tid, (uint64_t)B * H);
    float tc = tanhf(c_t[tid]);
    float d_o = dh * tc;
    float dcc = dc[tid] + dh * o * (1.f - tc * tc);
    float d_i = dcc * g, d_g = dcc * i, d_f = dcc * c_prev[tid];
    dc[tid] = dcc * f;
    float gi = d_i * i * (1.f - i), gf = d_f * f * (1.f - f), gg = d_g * (1.f - g * g), go = d_o * o * (1.f - o);
    float* drow = dG + (int64_t)b * 4 * H;
    drow[j] = gi; drow[H + j] = gf; drow[2 * H + j] = gg; drow[3 * H + j] = go;
    __half* hrow = dG_h + (int64_t)b * ld_g;
    hrow[j] = to_half_scaled(gi); hrow[H + j] = to_half_scaled(gf);
    hrow[2 * H + j] = to_half_scaled(gg); hrow[3 * H + j] = to_half_scaled(go);
}

int lstm_cell_bwd_tc(const float* dy_post, const float* dh_rec, float* dc, const float* gates, const float* c_t,
                     const float* c_prev, float* dG, __half* dG_h, int64_t ld_g, int B, int H, int64_t elem_off,
                     int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s, const float* r) {
    int64_t n = (int64_t)B * H;
    lstm_cell_bwd_tc_kernel<<<cdiv(n, 256), 256, 0, s>>>(dy_post, dh_rec, dc, gates, c_t, c_prev, dG, dG_h, ld_g, B, H,
                                                         elem_off, n_total, m, rm, r);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
