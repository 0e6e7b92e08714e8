// Pointwise kernels of the tensor-core engine: the cell rule of lstm_cell.cuh, as in pointwise.cu, plus the fp16 operand
// images the tensor-core GEMMs consume (h_t for the next step / wgrad, dropout(h_t) for the next
// layer, scaled dG and dS).  HBM/L2-bound, fully coalesced.
#include "lstm_cell.cuh"

namespace zrb {

// ZO: zoneout (DESIGN.md section 20), with h_{t-1} from h_prev and c~_t into c_til
template <bool ZO>
__global__ void lstm_cell_fwd_tc_kernel(float* __restrict__ pre, const float* __restrict__ c_prev,
                                        float* __restrict__ c_out, float* __restrict__ h_raw,
                                        __half* __restrict__ h_raw_h, __half* __restrict__ y_h, int64_t ld_h, int B,
                                        int H, int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm, ZoneoutSrc zo,
                                        const float* __restrict__ h_prev, float* __restrict__ c_til) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (int64_t)B * H) return;
    int b = (int)(tid / H), j = (int)(tid % H);
    float* row = pre + (int64_t)b * 4 * H;
    const uint32_t z = ZO && zo.flags ? zo.flags[elem_off + tid] : 0u;
    const CellFwd cf = cell_fwd<PreciseAct, ZO>(row[j], row[H + j], row[2 * H + j], row[3 * H + j], c_prev[tid],
                                                ZO ? h_prev[tid] : 0.f, z & 1u, z & 2u, zo);
    if constexpr (ZO) c_til[tid] = cf.ctil;
    row[j] = cf.i; row[H + j] = cf.f; row[2 * H + j] = cf.g; row[3 * H + j] = cf.o;
    c_out[tid] = cf.c;
    h_raw[tid] = cf.h;
    h_raw_h[(int64_t)b * ld_h + j] = __float2half_rn(cf.h * mask_mul1_at(rm, (uint64_t)tid, (uint64_t)B * H));   // next step's operand
    y_h[(int64_t)b * ld_h + j] = __float2half_rn(cf.h * mask_mul1(m, (uint64_t)(elem_off + tid), (uint64_t)n_total));
}

int lstm_cell_fwd_tc(float* pre, const float* c_prev, float* c_out, float* h_raw, __half* h_raw_h, __half* y_h,
                     int64_t ld_h, int B, int H, int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s,
                     const ZoneoutSrc* zo, const float* h_prev, float* c_til) {
    int64_t n = (int64_t)B * H;
    if (zo)
        lstm_cell_fwd_tc_kernel<true><<<cdiv(n, 256), 256, 0, s>>>(pre, c_prev, c_out, h_raw, h_raw_h, y_h, ld_h, B, H,
                                                                   elem_off, n_total, m, rm, *zo, h_prev, c_til);
    else
        lstm_cell_fwd_tc_kernel<false><<<cdiv(n, 256), 256, 0, s>>>(pre, c_prev, c_out, h_raw, h_raw_h, y_h, ld_h, B, H,
                                                                    elem_off, n_total, m, rm, ZoneoutSrc{}, nullptr,
                                                                    nullptr);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// ZO: c_t is c~_t, and hcarry [B,H] carries zh * dh from step t to step t-1 (the persistent kernel's register)
template <bool ZO>
__global__ void lstm_cell_bwd_tc_kernel(const float* __restrict__ dy_post, const float* __restrict__ dh_rec,
                                        float* __restrict__ dc, const float* __restrict__ gates,
                                        const float* __restrict__ c_t, const float* __restrict__ c_prev,
                                        float* __restrict__ dG, __half* __restrict__ dG_h, int64_t ld_g, int B, int H,
                                        int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm,
                                        const float* __restrict__ r, ZoneoutSrc zo, float* __restrict__ hcarry) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (int64_t)B * H) return;
    int b = (int)(tid / H), j = (int)(tid % H);
    const float* row = gates + (int64_t)b * 4 * H;
    const float i = row[j], f = row[H + j], g = row[2 * H + j], o = row[3 * H + j];
    float dh = dy_post[tid] * mask_mul1(m, (uint64_t)(elem_off + tid), (uint64_t)n_total);
    if (r) dh += r[tid];
    if (dh_rec) dh += dh_rec[tid] * mask_mul1_at(rm, (uint64_t)tid, (uint64_t)B * H);
    if constexpr (ZO) dh += hcarry[tid];
    const uint32_t z = ZO && zo.flags ? zo.flags[elem_off + tid] : 0u;
    float unused;
    const CellGrad d = cell_bwd<PreciseAct, ZO>(i, f, g, o, c_t[tid], c_prev[tid], dh, dc[tid], ZO ? hcarry[tid] : unused,
                                                z & 1u, z & 2u, zo);
    float* drow = dG + (int64_t)b * 4 * H;
    drow[j] = d.i; drow[H + j] = d.f; drow[2 * H + j] = d.g; drow[3 * H + j] = d.o;
    __half* hrow = dG_h + (int64_t)b * ld_g;
    hrow[j] = f16_sat(d.i * kGradScale); hrow[H + j] = f16_sat(d.f * kGradScale);
    hrow[2 * H + j] = f16_sat(d.g * kGradScale); hrow[3 * H + j] = f16_sat(d.o * kGradScale);
}

int lstm_cell_bwd_tc(const float* dy_post, const float* dh_rec, float* dc, const float* gates, const float* c_t,
                     const float* c_prev, float* dG, __half* dG_h, int64_t ld_g, int B, int H, int64_t elem_off,
                     int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s, const float* r, const ZoneoutSrc* zo,
                     float* hcarry) {
    int64_t n = (int64_t)B * H;
    if (zo)
        lstm_cell_bwd_tc_kernel<true><<<cdiv(n, 256), 256, 0, s>>>(dy_post, dh_rec, dc, gates, c_t, c_prev, dG, dG_h, ld_g,
                                                                   B, H, elem_off, n_total, m, rm, r, *zo, hcarry);
    else
        lstm_cell_bwd_tc_kernel<false><<<cdiv(n, 256), 256, 0, s>>>(dy_post, dh_rec, dc, gates, c_t, c_prev, dG, dG_h,
                                                                    ld_g, B, H, elem_off, n_total, m, rm, r,
                                                                    ZoneoutSrc{}, nullptr);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

__global__ void zoneout_flags_kernel(MaskSrc c, MaskSrc h, int64_t n, uint8_t* __restrict__ flags) {
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; 4 * g < n; g += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t kc = c.active ? mask_keep4(c, (uint64_t)g, (uint64_t)n) : 0xFu;
        const uint32_t kh = h.active ? mask_keep4(h, (uint64_t)g, (uint64_t)n) : 0xFu;
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (4 * g + i < n) flags[4 * g + i] = (uint8_t)((~kc >> i & 1u) | (~kh >> i & 1u) << 1);
    }
}

int zoneout_flags(MaskSrc c, MaskSrc h, int64_t n, uint8_t* flags, cudaStream_t s) {
    const int64_t quads = (n + 3) / 4;
    const int blocks = (int)(quads < 4096 * 256 ? cdiv(quads, 256) : 4096);
    zoneout_flags_kernel<<<blocks > 0 ? blocks : 1, 256, 0, s>>>(c, h, n, flags);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
