// fp32 -> fp16 image builders for the tensor-core engine (HBM-bound streaming kernels).
#include "kernels.h"
#include "tc_kernels.h"

namespace zrb {

// dst[r, 0..cols) = half(scale * src[r, 0..cols)), dst pitch ld_dst (>= cols), pad columns zeroed.
// m active (weight drop, DESIGN.md section 15): dst[r, c] = half(scale * fp32(src[r, c] * mul(r*ld_src + c))), four
// consecutive columns per thread so that each quad of mask elements costs one Philox call (ld_dst % 4 == 0)
__global__ void convert_pad_kernel(const float* __restrict__ src, int64_t ld_src, __half* __restrict__ dst,
                                   int64_t ld_dst, int rows, int cols, float scale, MaskSrc m) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t total = (int64_t)rows * ld_dst;
    if (m.active) {
        for (i *= 4; i < total; i += (int64_t)gridDim.x * blockDim.x * 4) {
            const int r = (int)(i / ld_dst), c0 = (int)(i % ld_dst);
            float mul[4];
            mask_mul4_at(m, (uint64_t)r * ld_src + c0, mul);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                dst[i + k] = f16_sat(c0 + k < cols ? src[(int64_t)r * ld_src + c0 + k] * mul[k] * scale : 0.f);
            }
        }
        return;
    }
    for (; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int r = (int)(i / ld_dst), c = (int)(i % ld_dst);
        dst[i] = f16_sat(c < cols ? src[(int64_t)r * ld_src + c] * scale : 0.f);
    }
}

int convert_pad_f16(const float* src, int64_t ld_src, __half* dst, int64_t ld_dst, int rows, int cols, float scale,
                    cudaStream_t s, MaskSrc m) {
    int64_t total = (int64_t)rows * ld_dst;
    if (!total) return ZRB_OK;
    ZRB_REQUIRE(!m.active || (ld_dst % 4 == 0 && !m.explicit_mask), "masked convert_pad_f16 needs ld_dst %% 4 == 0");
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    convert_pad_kernel<<<blocks, 256, 0, s>>>(src, ld_src, dst, ld_dst, rows, cols, scale, m);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

__global__ void fwd_prep_kernel(FwdPrep a) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    for (int l = 0; l < a.L; ++l) {
        const int H = a.H[l], Hp = a.Hp[l], GB = a.GB[l];
        const int bh = a.B * H, bhp = a.B * Hp, img_n = a.Kc[l] * GB * 64;
        const float* __restrict__ h = a.in_h[l];
        const float* __restrict__ c = a.in_c[l];
        const MaskSrc rm = a.rm[l];   // variational mode: the recurrent operand of step 0 is h0 * rm
        for (int i = tid; i < bh; i += nth) {
            a.h0s[l][i] = h[i];
            a.c0s[l][i] = c[i];
        }
        for (int i = tid; i < bhp; i += nth) {
            const int r = i / Hp, col = i % Hp;
            a.hprev_h[l][i] = __float2half_rn(
                col < H ? h[(size_t)r * H + col] * mask_mul1_at(rm, (uint64_t)r * H + col, (uint64_t)bh) : 0.f);
        }
        if (a.h0_img[l]) {
            for (int i = tid; i < img_n; i += nth) {
                const int e = i & 7, r = (i >> 3) & 7, g = (i >> 6) % GB, kc = (i >> 6) / GB;
                const int b = g * 8 + r, k = kc * 8 + e;
                a.h0_img[l][i] = __float2half_rn(
                    (b < a.B && k < H) ? h[(size_t)b * H + k] * mask_mul1_at(rm, (uint64_t)b * H + k, (uint64_t)bh) : 0.f);
            }
        }
    }
    for (int i = tid; i < a.N; i += nth) a.x_saved[i] = a.x[i];
}
int fwd_prep(const FwdPrep& a, cudaStream_t s) {
    int work = a.N;
    for (int l = 0; l < a.L; ++l) work = max(work, max(a.B * a.Hp[l], a.Kc[l] * a.GB[l] * 64));
    int blocks = cdiv(work, 256);
    if (blocks > 132 * 2) blocks = 132 * 2;
    if (blocks < 1) blocks = 1;
    fwd_prep_kernel<<<blocks, 256, 0, s>>>(a);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// out[j] = inv_scale * sum_n A[n, j]  for an fp16 matrix with pitch ld (bias gradients: column sums of dG / dS).
// Pass 1: block (x, y) owns 64 columns and every kRowSplit-th slab of rows (16 row-lanes, one __half2 per
// thread) and writes a partial; pass 2 adds the kRowSplit partials in fixed order (deterministic).
constexpr int kRowSplit = 8;
__global__ void colsum_h_partial_kernel(const __half* __restrict__ A, int64_t ld, float* __restrict__ part_out, int N,
                                        int M, int Mp) {
    __shared__ float part[16][65];
    const int col = blockIdx.x * 64 + threadIdx.x * 2;
    const int rows_per = (N + kRowSplit - 1) / kRowSplit;
    const int n0 = blockIdx.y * rows_per, n1 = min(N, n0 + rows_per);
    float a0 = 0.f, a1 = 0.f;
    if (col < M) {   // the pitch is even and >= M, so the __half2 read stays inside the row
#pragma unroll 4
        for (int n = n0 + threadIdx.y; n < n1; n += 16) {
            __half2 v = *reinterpret_cast<const __half2*>(A + (int64_t)n * ld + col);
            a0 += __low2float(v);
            a1 += __high2float(v);
        }
    }
    part[threadIdx.y][threadIdx.x * 2] = a0;
    part[threadIdx.y][threadIdx.x * 2 + 1] = a1;
    __syncthreads();
    const int t = threadIdx.y * 32 + threadIdx.x;
    if (t < 64 && blockIdx.x * 64 + t < M) {
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < 16; ++r) s += part[r][t];
        part_out[(int64_t)blockIdx.y * Mp + blockIdx.x * 64 + t] = s;
    }
}
__global__ void colsum_h_final_kernel(const float* __restrict__ part, float* __restrict__ out, float* __restrict__ out2,
                                      int M, int Mp, float inv_scale) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= M) return;
    float s = 0.f;
#pragma unroll
    for (int y = 0; y < kRowSplit; ++y) s += part[(int64_t)y * Mp + j];
    out[j] = s * inv_scale;
    if (out2) out2[j] = s * inv_scale;
}
int colsum_h_scratch_floats(int M) { return kRowSplit * ((M + 63) / 64 * 64); }

// scratch: colsum_h_scratch_floats(M) floats owned by the caller's context (per device, per stream of use)
int colsum_h(const __half* A, int64_t ld, float* out, float* out2, int N, int M, float inv_scale, float* scratch,
             cudaStream_t s) {
    const int Mp = (M + 63) / 64 * 64;
    dim3 blk(32, 16), grid(Mp / 64, kRowSplit);
    colsum_h_partial_kernel<<<grid, blk, 0, s>>>(A, ld, scratch, N, M, Mp);
    ZRB_KERNEL_CHECK();
    colsum_h_final_kernel<<<cdiv(M, 256), 256, 0, s>>>(scratch, out, out2, M, Mp, inv_scale);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
