// HBM-bound kernels of the path: embedding gather/scatter, dropout, LSTM cell pointwise
// math (validation engine), bias/column sums, softmax-NLL.  Coalesced row-major access;
// no tensor-core work here.
#include "kernels.h"
#include "lstm_cell.cuh"

namespace zrb {

// ----------------------------------------------------------------------------------------
// Embedding gather fused with the first dropout site.   model.py:13-14, :105
// grid: one block per token row; threads stride the row in groups of 4 (one Philox call
// yields the keep flags of 4 consecutive elements).
// Algorithmic bytes per token: H*4 read (table row) + H*4 written (+ H*2 fp16 image).
// PENDING (tied embedding, lazy update): the SGD update of W is still deferred; every gathered element is
// sgd_elem(W, coef * g, lr) with the coefficient of scalars[1], the value update_pack will store (g is only read).
// em: embedding dropout (DESIGN.md section 17), one keep flag per vocabulary row; the row is multiplied by its
// multiplier s_e before the site-0 mask: fp32(fp32(W * s_e) * s_0).  One Philox call per thread (the whole row
// shares the flag), none when inactive.
// ----------------------------------------------------------------------------------------
template <bool PENDING>
__global__ void embed_dropout_fwd_kernel(const float* __restrict__ W, const int64_t* __restrict__ idx,
                                         float* __restrict__ out, __half* __restrict__ out_h, int64_t ld_h, int N,
                                         int H, int V, MaskSrc m, MaskSrc em, const float* __restrict__ pend_g, float lr,
                                         const float* __restrict__ scalars) {
    int n = blockIdx.x;
    if (n >= N) return;
    int64_t row = idx[n];
    if (row < 0 || row >= V) row = 0;  // the reference would raise; never dereference OOB
    const float* src = W + row * (int64_t)H;
    int groups = (H + 3) >> 2;
    uint64_t n_total = (uint64_t)N * H;
    float coef = 0.f;
    if constexpr (PENDING) coef = scalars[1];
    const float se = em.active ? mask_mul1_at(em, (uint64_t)row, (uint64_t)V) : 1.f;
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
        int j0 = g << 2;
        uint64_t e0 = (uint64_t)n * H + j0;
        float v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if constexpr (PENDING) v[i] = (j0 + i < H) ? sgd_elem(src[j0 + i], pend_g[row * (int64_t)H + j0 + i] * coef, lr) : 0.f;
            else v[i] = (j0 + i < H) ? src[j0 + i] : 0.f;
        }
        if (em.active) {
#pragma unroll
            for (int i = 0; i < 4; ++i) v[i] *= se;
        }
        if (m.active) {
            // rows are H long; H % 4 != 0 makes groups straddle Philox quads -> per-element path.  (A variational
            // period B*H is then a multiple of 4 too, so the reduced e0 still starts a quad.)
            if ((H & 3) == 0) {
                uint32_t bits = mask_keep4(m, mask_elem(m, e0) >> 2, n_total);
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = ((bits >> i) & 1u) ? v[i] * m.scale : 0.f;
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] *= mask_mul1(m, e0 + i, n_total);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (j0 + i < H) {
                if (out) out[(int64_t)n * H + j0 + i] = v[i];
                if (out_h) out_h[(int64_t)n * ld_h + j0 + i] = __float2half_rn(v[i]);
            }
        }
    }
}

int embed_dropout_fwd(const float* W, const int64_t* idx, float* out, __half* out_h, int64_t ld_h, int N, int H,
                      int V, MaskSrc m, MaskSrc em, cudaStream_t s, const float* pend_g, float lr, const float* scalars) {
    if (N == 0) return ZRB_OK;
    int threads = H >= 1024 ? 256 : 128;
    if (pend_g) embed_dropout_fwd_kernel<true><<<N, threads, 0, s>>>(W, idx, out, out_h, ld_h, N, H, V, m, em, pend_g, lr, scalars);
    else embed_dropout_fwd_kernel<false><<<N, threads, 0, s>>>(W, idx, out, out_h, ld_h, N, H, V, m, em, nullptr, 0.f, nullptr);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// Backward of the gather: scatter-add with fp32 atomics (duplicate tokens in a window hit
// the same row).  dW must be zeroed by the caller.  Each occurrence adds fp32(fp32(dA * s_0) * s_e).
__global__ void embed_dropout_bwd_kernel(const float* __restrict__ dA, const int64_t* __restrict__ idx,
                                         float* __restrict__ dW, int N, int H, int V, MaskSrc m, MaskSrc em) {
    int n = blockIdx.x;
    if (n >= N) return;
    int64_t row = idx[n];
    if (row < 0 || row >= V) return;
    uint64_t n_total = (uint64_t)N * H;
    const float se = em.active ? mask_mul1_at(em, (uint64_t)row, (uint64_t)V) : 1.f;
    for (int j = threadIdx.x; j < H; j += blockDim.x) {
        float g = dA[(int64_t)n * H + j] * mask_mul1(m, (uint64_t)n * H + j, n_total);
        if (em.active) g *= se;
        if (g != 0.f) atomicAdd(dW + row * (int64_t)H + j, g);
    }
}

int embed_dropout_bwd(const float* dA, const int64_t* idx, float* dW, int N, int H, int V, MaskSrc m, MaskSrc em,
                      cudaStream_t s) {
    if (N == 0) return ZRB_OK;
    embed_dropout_bwd_kernel<<<N, 256, 0, s>>>(dA, idx, dW, N, H, V, m, em);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// ----------------------------------------------------------------------------------------
// LSTM cell pointwise (validation engine): the cell rule of lstm_cell.cuh with expf / tanhf.
// ----------------------------------------------------------------------------------------
__global__ void lstm_cell_fwd_kernel(float* __restrict__ pre, const float* __restrict__ c_prev,
                                     float* __restrict__ c_out, float* __restrict__ h_raw, float* __restrict__ y_out,
                                     float* __restrict__ h_rec, int B, int H, int64_t elem_off, int64_t n_total, MaskSrc m,
                                     MaskSrc rm) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (int64_t)B * H) return;
    int b = (int)(tid / H), j = (int)(tid % H);
    float* row = pre + (int64_t)b * 4 * H;
    const CellFwd cf = cell_fwd<PreciseAct, false>(row[j], row[H + j], row[2 * H + j], row[3 * H + j], c_prev[tid], 0.f,
                                                   false, false, ZoneoutSrc{});
    row[j] = cf.i; row[H + j] = cf.f; row[2 * H + j] = cf.g; row[3 * H + j] = cf.o;
    c_out[tid] = cf.c;
    h_raw[tid] = cf.h;
    y_out[tid] = cf.h * mask_mul1(m, (uint64_t)(elem_off + tid), (uint64_t)n_total);
    if (h_rec) h_rec[tid] = cf.h * mask_mul1_at(rm, (uint64_t)tid, (uint64_t)B * H);   // the next step's recurrent operand
}

int lstm_cell_fwd(float* pre, const float* c_prev, float* c_out, float* h_raw, float* y_out, float* h_rec, int B, int H,
                  int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s) {
    int64_t n = (int64_t)B * H;
    lstm_cell_fwd_kernel<<<cdiv(n, 256), 256, 0, s>>>(pre, c_prev, c_out, h_raw, y_out, h_rec, B, H, elem_off, n_total, m,
                                                      rm);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// SURVEY 8a backward: dh = mask*dy + dh_rec, then the cell rule
__global__ void lstm_cell_bwd_kernel(const float* __restrict__ dy_post, const float* __restrict__ dh_rec,
                                     float* __restrict__ dc, const float* __restrict__ gates,
                                     const float* __restrict__ c_t, const float* __restrict__ c_prev,
                                     float* __restrict__ dG, int B, int H, int64_t elem_off, int64_t n_total,
                                     MaskSrc m, MaskSrc rm, const float* __restrict__ r) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (int64_t)B * H) return;
    int b = (int)(tid / H), j = (int)(tid % H);
    const float* row = gates + (int64_t)b * 4 * H;
    const float i = row[j], f = row[H + j], g = row[2 * H + j], o = row[3 * H + j];
    float dh = dy_post[tid] * mask_mul1(m, (uint64_t)(elem_off + tid), (uint64_t)n_total);
    if (r) dh += r[tid];
    if (dh_rec) dh += dh_rec[tid] * mask_mul1_at(rm, (uint64_t)tid, (uint64_t)B * H);
    float unused;
    const CellGrad d = cell_bwd<PreciseAct, false>(i, f, g, o, c_t[tid], c_prev[tid], dh, dc[tid], unused, false, false,
                                                   ZoneoutSrc{});
    float* drow = dG + (int64_t)b * 4 * H;
    drow[j] = d.i; drow[H + j] = d.f; drow[2 * H + j] = d.g; drow[3 * H + j] = d.o;
}

int lstm_cell_bwd(const float* dy_post, const float* dh_rec, float* dc, const float* gates, const float* c_t,
                  const float* c_prev, float* dG, int B, int H, int64_t elem_off, int64_t n_total, MaskSrc m,
                  MaskSrc rm, cudaStream_t s, const float* r) {
    int64_t n = (int64_t)B * H;
    lstm_cell_bwd_kernel<<<cdiv(n, 256), 256, 0, s>>>(dy_post, dh_rec, dc, gates, c_t, c_prev, dG, B, H, elem_off,
                                                      n_total, m, rm, r);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// ---- AR / TAR (DESIGN.md section 17) ------------------------------------------------------------------------------
// Over the last layer's raw output h [T, B*H] (bh = B*H), with s = the output site's multiplier of element e:
//   y = fp32(h * s);  dp = h_t - h_{t-1} (t >= 1, else 0);  dn = h_{t+1} - h_t (t <= T-2, else 0)
//   r = fp32(fp32(ca * y) * s) + fp32(cb * fp32(dp - dn))
// and, per block (fixed grid, fixed block size, fixed tree: a step stays reproducible), the fp64 sums of y^2 and dp^2.
__global__ void __launch_bounds__(256) act_reg_kernel(const float* __restrict__ h, float* __restrict__ r,
                                                      double* __restrict__ partial, int T, int64_t bh, MaskSrc m,
                                                      float ca, float cb) {
    const int64_t n = (int64_t)T * bh;
    double sy = 0.0, sd = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(e / bh);
        const float hv = h[e];
        const float s = mask_mul1(m, (uint64_t)e, (uint64_t)n);
        const float y = __fmul_rn(hv, s);
        const float dp = t > 0 ? __fsub_rn(hv, h[e - bh]) : 0.f;
        const float dn = t < T - 1 ? __fsub_rn(h[e + bh], hv) : 0.f;
        r[e] = __fadd_rn(__fmul_rn(__fmul_rn(ca, y), s), __fmul_rn(cb, __fsub_rn(dp, dn)));   // (no contraction)
        sy += (double)y * y;
        sd += (double)dp * dp;
    }
    __shared__ double red[2][8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
        sd += __shfl_xor_sync(0xffffffffu, sd, o);
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = sy; red[1][threadIdx.x >> 5] = sd; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int w = 0; w < 8; ++w) { a += red[0][w]; b += red[1][w]; }
        partial[2 * blockIdx.x] = a;
        partial[2 * blockIdx.x + 1] = b;
    }
}

// out[0] = fp32(wa * sum y^2), out[1] = fp32(wb * sum dp^2), the partials added in block order
__global__ void act_reg_finish_kernel(const double* __restrict__ partial, int nblocks, double wa, double wb,
                                      float* __restrict__ out) {
    if (threadIdx.x != 0) return;
    double a = 0.0, b = 0.0;
    for (int i = 0; i < nblocks; ++i) { a += partial[2 * i]; b += partial[2 * i + 1]; }
    out[0] = (float)(wa * a);
    out[1] = (float)(wb * b);
}

int activation_reg(const float* h, float* r, double* partial, float* out, int T, int B, int H, MaskSrc m, float alpha,
                   float beta, cudaStream_t s) {
    const int64_t bh = (int64_t)B * H;
    const double wa = (double)alpha / ((double)T * H);
    const double wb = T > 1 ? (double)beta / ((double)(T - 1) * H) : 0.0;
    act_reg_kernel<<<kActRegBlocks, 256, 0, s>>>(h, r, partial, T, bh, m, (float)(2.0 * wa), (float)(2.0 * wb));
    ZRB_KERNEL_CHECK();
    act_reg_finish_kernel<<<1, 32, 0, s>>>(partial, kActRegBlocks, wa, wb, out);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// y[e] = x[e] * mask multiplier of element e, e < n (the masked state entering the window, variational mode)
__global__ void dropout_copy_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t n, MaskSrc m) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n) y[e] = x[e] * mask_mul1(m, (uint64_t)e, (uint64_t)n);
}
int dropout_copy(const float* x, float* y, int64_t n, MaskSrc m, cudaStream_t s) {
    if (n == 0) return ZRB_OK;
    dropout_copy_kernel<<<cdiv(n, 256), 256, 0, s>>>(x, y, n, m);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// Weight drop (DESIGN.md section 15): y[e] = x[e] * mul(e) over n4 quads, one Philox call per quad; x may be y (the
// gradient pass, in place).  sumsq (or null): block b writes the sum of y^2 over its grid-stride share to sumsq[b], a
// fixed summation order, so the clip norm does not re-read the gradient.
__global__ void __launch_bounds__(256) weight_drop_kernel(const float* x, float* y, int64_t n4, MaskSrc m,
                                                          float* __restrict__ sumsq) {
    __shared__ float sh[8];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const bool vec = ((((uintptr_t)x) | ((uintptr_t)y)) & 15) == 0;
    float acc = 0.f;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += stride) {
        float mul[4];
        mask_mul4_at(m, (uint64_t)q * 4, mul);
        float4 v;
        if (vec) {
            v = reinterpret_cast<const float4*>(x)[q];
        } else {
            v.x = x[4 * q]; v.y = x[4 * q + 1]; v.z = x[4 * q + 2]; v.w = x[4 * q + 3];
        }
        v.x *= mul[0]; v.y *= mul[1]; v.z *= mul[2]; v.w *= mul[3];
        if (vec) {
            reinterpret_cast<float4*>(y)[q] = v;
        } else {
            y[4 * q] = v.x; y[4 * q + 1] = v.y; y[4 * q + 2] = v.z; y[4 * q + 3] = v.w;
        }
        acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    if (!sumsq) return;
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += sh[w];
        sumsq[blockIdx.x] = t;
    }
}
int weight_drop(const float* x, float* y, int64_t n, MaskSrc m, float* sumsq, cudaStream_t s) {
    ZRB_REQUIRE(n % 4 == 0 && !m.explicit_mask, "weight_drop: n=%lld must be a multiple of 4", (long long)n);
    weight_drop_kernel<<<kWeightDropBlocks, 256, 0, s>>>(x, y, n / 4, m, sumsq);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// ----------------------------------------------------------------------------------------
__global__ void add_bias_kernel(float* __restrict__ C, const float* __restrict__ b1, const float* __restrict__ b2,
                                int64_t total, int M) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int j = (int)(i % M);
    float v = b1[j];
    if (b2) v += b2[j];
    C[i] += v;
}
int add_bias2(float* C, const float* b1, const float* b2, int N, int M, cudaStream_t s) {
    int64_t total = (int64_t)N * M;
    if (!total) return ZRB_OK;
    add_bias_kernel<<<cdiv(total, 256), 256, 0, s>>>(C, b1, b2, total, M);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}
int add_bias1(float* C, const float* b1, int N, int M, cudaStream_t s) { return add_bias2(C, b1, nullptr, N, M, s); }

// out[j] = sum_n A[n,j]: a block owns 32 columns; 8 row-lanes stride the rows, then a
// shared-memory tree over the 8 partials (deterministic).
__global__ void colsum_kernel(const float* __restrict__ A, float* __restrict__ out, float* __restrict__ out2, int N,
                              int M) {
    __shared__ float part[8][33];
    int col = blockIdx.x * 32 + threadIdx.x;
    float acc = 0.f;
    if (col < M)
        for (int n = threadIdx.y; n < N; n += 8) acc += A[(int64_t)n * M + col];
    part[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && col < M) {
        float t = 0.f;
#pragma unroll
        for (int r = 0; r < 8; ++r) t += part[r][threadIdx.x];
        out[col] = t;
        if (out2) out2[col] = t;
    }
}
int colsum(const float* A, float* out, float* out2, int N, int M, cudaStream_t s) {
    dim3 blk(32, 8);
    colsum_kernel<<<cdiv(M, 32), blk, 0, s>>>(A, out, out2, N, M);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// ----------------------------------------------------------------------------------------
// softmax-NLL forward (+ gradient) -- main.py:77-84.  One block per token row; the row is
// read twice from L2/HBM (max+sum pass fused as online softmax, then the write pass).
// The reference exponentiates without subtracting the max (overflows beyond ~88); the
// max-subtracted form is the same function where the reference is finite.
// Algorithmic bytes per token: V*4 read + V*4 written (dscores).
// ----------------------------------------------------------------------------------------
__global__ void softmax_nll_kernel(const float* __restrict__ scores, const int64_t* __restrict__ y, int N, int V,
                                   float gscale, float* __restrict__ row_loss, float* __restrict__ dscores,
                                   float* __restrict__ tgt_prob, __half* __restrict__ ds_h, int64_t ld_s,
                                   float h_scale) {
    __shared__ float s_m[32], s_s[32];
    int n = blockIdx.x;
    const float* row = scores + (int64_t)n * V;
    float mx = -INFINITY, sum = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        float z = row[v];
        if (z > mx) {
            sum = sum * __expf(mx - z) + 1.f;
            mx = z;
        } else {
            sum += __expf(z - mx);
        }
    }
    // warp then block combine of (max, sum) pairs
    for (int o = 16; o > 0; o >>= 1) {
        float om = __shfl_xor_sync(0xffffffffu, mx, o);
        float os = __shfl_xor_sync(0xffffffffu, sum, o);
        float nm = fmaxf(mx, om);
        sum = (mx == -INFINITY ? 0.f : sum * __expf(mx - nm)) + (om == -INFINITY ? 0.f : os * __expf(om - nm));
        mx = nm;
    }
    int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (l == 0) { s_m[w] = mx; s_s[w] = sum; }
    __syncthreads();
    if (w == 0) {
        mx = l < nw ? s_m[l] : -INFINITY;
        sum = l < nw ? s_s[l] : 0.f;
        for (int o = 16; o > 0; o >>= 1) {
            float om = __shfl_xor_sync(0xffffffffu, mx, o);
            float os = __shfl_xor_sync(0xffffffffu, sum, o);
            float nm = fmaxf(mx, om);
            sum = (mx == -INFINITY ? 0.f : sum * __expf(mx - nm)) + (om == -INFINITY ? 0.f : os * __expf(om - nm));
            mx = nm;
        }
        if (l == 0) { s_m[0] = mx; s_s[0] = sum; }
    }
    __syncthreads();
    mx = s_m[0];
    sum = s_s[0];
    int64_t tgt = y[n];
    float inv = 1.f / sum;
    if (threadIdx.x == 0) {
        float zt = (tgt >= 0 && tgt < V) ? row[tgt] : mx;
        row_loss[n] = -(zt - mx - logf(sum));
        if (tgt_prob) tgt_prob[n] = expf(zt - mx) * inv;
    }
    if (dscores || ds_h) {
        float* drow = dscores ? dscores + (int64_t)n * V : nullptr;
        __half* hrow = ds_h ? ds_h + (int64_t)n * ld_s : nullptr;
        for (int v = threadIdx.x; v < V; v += blockDim.x) {
            float p = __expf(row[v] - mx) * inv;
            if (v == tgt) p -= 1.f;
            p *= gscale;
            if (drow) drow[v] = p;
            if (hrow) hrow[v] = f16_sat(p * h_scale);
        }
    }
}

// Same function with the row held in registers: one block per token, every thread loads NV float4 chunks ONCE
// (the scalar kernel above reads the row twice and carries the online-softmax recurrence through every element),
// block max, one exp per element, block sum, then the gradient is written from the registers with 16-byte
// (fp32) / 8-byte (fp16 image) stores.  Needs V % 4 == 0, V <= 4 * 512 * NV and 16-byte aligned rows.
constexpr int kSmThreads = 512;
__device__ __forceinline__ float block_reduce_512(float v, float* sh, bool is_max) {
    for (int o = 16; o > 0; o >>= 1) {
        float t = __shfl_xor_sync(0xffffffffu, v, o);
        v = is_max ? fmaxf(v, t) : v + t;
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();                       // sh may still be read from the previous reduction
    if (l == 0) sh[w] = v;
    __syncthreads();
    v = l < kSmThreads / 32 ? sh[l] : (is_max ? -INFINITY : 0.f);
    for (int o = 16; o > 0; o >>= 1) {
        float t = __shfl_xor_sync(0xffffffffu, v, o);
        v = is_max ? fmaxf(v, t) : v + t;
    }
    return v;                              // every thread holds the block result (fixed tree: deterministic)
}
template <int NV>
__global__ void __launch_bounds__(kSmThreads) softmax_nll_reg_kernel(
    const float* __restrict__ scores, const int64_t* __restrict__ y, int N, int V, float gscale,
    float* __restrict__ row_loss, float* __restrict__ dscores, float* __restrict__ tgt_prob, __half* __restrict__ ds_h,
    int64_t ld_s, float h_scale) {
    __shared__ float sh[32];
    const int n = blockIdx.x;
    const float* row = scores + (int64_t)n * V;
    const float4* row4 = reinterpret_cast<const float4*>(row);
    const int nv4 = V >> 2;
    float4 z[NV];
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int i = threadIdx.x + k * kSmThreads;
        if (i < nv4) {
            z[k] = __ldcs(row4 + i);
            mx = fmaxf(mx, fmaxf(fmaxf(z[k].x, z[k].y), fmaxf(z[k].z, z[k].w)));
        }
    }
    mx = block_reduce_512(mx, sh, true);
    if (mx == -INFINITY) mx = 0.f;
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int i = threadIdx.x + k * kSmThreads;
        if (i < nv4) {
            z[k].x = __expf(z[k].x - mx); z[k].y = __expf(z[k].y - mx);
            z[k].z = __expf(z[k].z - mx); z[k].w = __expf(z[k].w - mx);
            sum += (z[k].x + z[k].y) + (z[k].z + z[k].w);
        }
    }
    sum = block_reduce_512(sum, sh, false);
    const float inv = 1.f / sum;
    const int64_t tgt = y[n];
    if (threadIdx.x == 0) {
        const float zt = (tgt >= 0 && tgt < V) ? row[tgt] : mx;
        row_loss[n] = -(zt - mx - logf(sum));
        if (tgt_prob) tgt_prob[n] = expf(zt - mx) * inv;
    }
    if (dscores || ds_h) {
        float4* drow = dscores ? reinterpret_cast<float4*>(dscores + (int64_t)n * V) : nullptr;
        uint2* hrow = ds_h ? reinterpret_cast<uint2*>(ds_h + (int64_t)n * ld_s) : nullptr;
        const float g = gscale * inv;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int i = threadIdx.x + k * kSmThreads;
            if (i < nv4) {
                float4 p = make_float4(z[k].x * g, z[k].y * g, z[k].z * g, z[k].w * g);
                const int64_t d = tgt - 4 * (int64_t)i;        // the target's position inside this chunk, if any
                if (d == 0) p.x -= gscale; else if (d == 1) p.y -= gscale; else if (d == 2) p.z -= gscale;
                else if (d == 3) p.w -= gscale;
                if (drow) drow[i] = p;
                if (hrow) {
                    const float lo = -65504.f, hi = 65504.f;
                    __half2 a = __floats2half2_rn(fminf(fmaxf(p.x * h_scale, lo), hi), fminf(fmaxf(p.y * h_scale, lo), hi));
                    __half2 b = __floats2half2_rn(fminf(fmaxf(p.z * h_scale, lo), hi), fminf(fmaxf(p.w * h_scale, lo), hi));
                    uint2 u;
                    u.x = *reinterpret_cast<uint32_t*>(&a);
                    u.y = *reinterpret_cast<uint32_t*>(&b);
                    hrow[i] = u;
                }
            }
        }
    }
}

// loss = (B / N) * sum_n row_loss[n]  (fixed-order tree: deterministic)
__global__ void loss_reduce_kernel(const float* __restrict__ row_loss, int N, float scale, float* __restrict__ loss) {
    __shared__ float sh[32];
    float acc = 0.f;
    for (int n = threadIdx.x; n < N; n += blockDim.x) acc += row_loss[n];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) *loss = v * scale;
    }
}

int softmax_nll(const float* scores, const int64_t* y, int N, int V, int B, float* row_loss, float* loss,
                float* dscores, float* tgt_prob, cudaStream_t s, __half* ds_h, int64_t ld_s, float h_scale) {
    if (N == 0) return ZRB_OK;
    float gscale = (float)((double)B / (double)N);
    const bool vec = V % 4 == 0 && V <= 4 * kSmThreads * 8 && (((uintptr_t)scores) & 15) == 0 &&
                     (!dscores || (((uintptr_t)dscores) & 15) == 0) &&
                     (!ds_h || ((((uintptr_t)ds_h) & 7) == 0 && ld_s % 4 == 0));
    const int nv = vec ? (V / 4 + kSmThreads - 1) / kSmThreads : 0;
#define ZRB_SM_LAUNCH(NV) \
    softmax_nll_reg_kernel<NV><<<N, kSmThreads, 0, s>>>(scores, y, N, V, gscale, row_loss, dscores, tgt_prob, ds_h, ld_s, h_scale)
    if (vec && nv <= 2) ZRB_SM_LAUNCH(2);
    else if (vec && nv <= 4) ZRB_SM_LAUNCH(4);
    else if (vec && nv <= 6) ZRB_SM_LAUNCH(6);
    else if (vec) ZRB_SM_LAUNCH(8);
    else softmax_nll_kernel<<<N, 512, 0, s>>>(scores, y, N, V, gscale, row_loss, dscores, tgt_prob, ds_h, ld_s, h_scale);
#undef ZRB_SM_LAUNCH
    ZRB_KERNEL_CHECK();
    if (loss) ZRB_TRY(loss_reduce(row_loss, N, gscale, loss, s));
    return ZRB_OK;
}

int loss_reduce(const float* row_loss, int N, float scale, float* loss, cudaStream_t s) {
    loss_reduce_kernel<<<1, 256, 0, s>>>(row_loss, N, scale, loss);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// ---- sparse form of the embedding gradient (data parallel) ------------------------------------------------
// rows[n, :] = dropout-masked dA[n, :]: what embed_dropout_bwd would scatter, kept as N rows so that ranks can
// exchange 4 MB of rows instead of all-reducing the dense 60 MB table gradient.  Embedding dropout (em active): row n
// is fp32(fp32(dA * s_0) * s_e) with the flag of its token idx[n], so the rows leave the library already masked.
__global__ void embed_rows_kernel(const float* __restrict__ dA, const int64_t* __restrict__ idx, float* __restrict__ rows,
                                  int N, int H, int V, MaskSrc m, MaskSrc em) {
    int n = blockIdx.x;
    uint64_t n_total = (uint64_t)N * H;
    float se = 1.f;
    if (em.active) {
        const int64_t row = idx[n];
        se = (row >= 0 && row < V) ? mask_mul1_at(em, (uint64_t)row, (uint64_t)V) : 0.f;   // (the scatter skips it)
    }
    for (int j = threadIdx.x; j < H; j += blockDim.x) {
        float g = dA[(int64_t)n * H + j] * mask_mul1(m, (uint64_t)n * H + j, n_total);
        if (em.active) g *= se;
        rows[(int64_t)n * H + j] = g;
    }
}
int embed_rows(const float* dA, const int64_t* idx, float* rows, int N, int H, int V, MaskSrc m, MaskSrc em,
               cudaStream_t s) {
    if (!N) return ZRB_OK;
    embed_rows_kernel<<<N, 256, 0, s>>>(dA, idx, rows, N, H, V, m, em);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// dW[id, :] = sum of rows[n, :] over all n with ids[n] == id, bit-identical on every rank that holds the same
// (ids, rows) arrays: the rows are accumulated as 64-bit fixed point (2^-40 resolution, |x| < 8e6) with integer
// atomics, whose result does not depend on the order of the additions, into the slot of the id's first
// occurrence (atomicMin), then converted back to fp32 once.
__global__ void embed_first_kernel(const int64_t* __restrict__ ids, int* __restrict__ first, int n_rows, int V) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_rows) return;
    int64_t id = ids[n];
    if (id >= 0 && id < V) atomicMin(first + id, n);
}
__global__ void embed_accum_kernel(const int64_t* __restrict__ ids, const float* __restrict__ rows,
                                   const int* __restrict__ first, long long* __restrict__ acc, int n_rows, int H, int V) {
    const int n = blockIdx.x;
    const int64_t id = ids[n];
    if (id < 0 || id >= V) return;
    long long* dst = acc + (int64_t)first[id] * H;
    for (int j = threadIdx.x; j < H; j += blockDim.x) {
        float v = rows[(int64_t)n * H + j];
        if (v != 0.f) atomicAdd((unsigned long long*)(dst + j), (unsigned long long)__float2ll_rn(v * 1099511627776.f));
    }
}
__global__ void embed_finish_kernel(const int64_t* __restrict__ ids, const int* __restrict__ first,
                                    const long long* __restrict__ acc, float* __restrict__ dW, int n_rows, int H, int V) {
    const int n = blockIdx.x;
    const int64_t id = ids[n];
    if (id < 0 || id >= V || first[id] != n) return;
    for (int j = threadIdx.x; j < H; j += blockDim.x)
        dW[id * (int64_t)H + j] = (float)((double)acc[(int64_t)n * H + j] * (1.0 / 1099511627776.0));
}
// Tied embedding (DESIGN.md section 13): dW already holds the projection's weight gradient G; the id's sum e is added,
// dW[id] = fp32(G[id] + e).  sumsq (or null): the `nblocks` blocks grid-stride over the tokens and block k writes
// sumsq[k] = sum over its distinct ids' elements of (new^2 - old^2), so that a clip norm whose matrix part came from
// sums of squares of G (the wgrad GEMM epilogues) becomes that of the merged gradient without reading it again.
__global__ void embed_finish_add_kernel(const int64_t* __restrict__ ids, const int* __restrict__ first,
                                        const long long* __restrict__ acc, float* __restrict__ dW, int n_rows, int H,
                                        int V, float* __restrict__ sumsq) {
    __shared__ double sh[8];
    // new^2 - old^2 cancels in part when |e| << |G|: the squares of two fp32 values are exact in fp64 and the sum is
    // kept there, so the correction's error is one fp32 rounding of each block's total, not one per element
    double ss = 0.0;
    for (int n = blockIdx.x; n < n_rows; n += gridDim.x) {
        const int64_t id = ids[n];
        if (id < 0 || id >= V || first[id] != n) continue;
        for (int j = threadIdx.x; j < H; j += blockDim.x) {
            const float old = dW[id * (int64_t)H + j];
            const float e = (float)((double)acc[(int64_t)n * H + j] * (1.0 / 1099511627776.0));
            const float nw = old + e;
            dW[id * (int64_t)H + j] = nw;
            ss += (double)nw * nw - (double)old * old;
        }
    }
    if (!sumsq) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sh[i];
        sumsq[blockIdx.x] = (float)t;
    }
}
int embed_scatter_rows(const int64_t* ids, const float* rows, float* dW, int n_rows, int H, int V, int* first,
                       long long* acc, cudaStream_t s, bool add, float* sumsq, int nblocks) {
    if (!n_rows) return ZRB_OK;
    ZRB_CUDA(cudaMemsetAsync(first, 0x7f, (size_t)V * sizeof(int), s));           // 0x7f7f7f7f > any row index
    ZRB_CUDA(cudaMemsetAsync(acc, 0, (size_t)n_rows * H * sizeof(long long), s));
    embed_first_kernel<<<cdiv(n_rows, 256), 256, 0, s>>>(ids, first, n_rows, V);
    ZRB_KERNEL_CHECK();
    embed_accum_kernel<<<n_rows, 256, 0, s>>>(ids, rows, first, acc, n_rows, H, V);
    ZRB_KERNEL_CHECK();
    if (add) embed_finish_add_kernel<<<sumsq ? nblocks : n_rows, 256, 0, s>>>(ids, first, acc, dW, n_rows, H, V, sumsq);
    else embed_finish_kernel<<<n_rows, 256, 0, s>>>(ids, first, acc, dW, n_rows, H, V);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// ---- touched-rows-only handling of the embedding gradient (single process) ---------------------------------
// The dense [V,H] gradient is non-zero only in the <= N rows of this window's tokens.  Instead of zero-filling,
// norm-reading and updating 60 MB per step, only those rows are touched: rows of the PREVIOUS step are cleared,
// the first occurrence of every id (atomicMin table) owns the row for the norm and the update.
__global__ void embed_zero_rows_kernel(float* __restrict__ dW, const int64_t* __restrict__ ids, int n, int H, int V) {
    const int64_t id = ids[blockIdx.x];
    if (id < 0 || id >= V) return;
    for (int j = threadIdx.x; j < H; j += blockDim.x) dW[id * (int64_t)H + j] = 0.f;
}
int embed_zero_rows(float* dW, const int64_t* ids, int n, int H, int V, cudaStream_t s) {
    if (!n) return ZRB_OK;
    embed_zero_rows_kernel<<<n, 256, 0, s>>>(dW, ids, n, H, V);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}
int embed_first_table(const int64_t* ids, int* first, int n, int V, cudaStream_t s) {
    ZRB_CUDA(cudaMemsetAsync(first, 0x7f, (size_t)V * sizeof(int), s));
    if (!n) return ZRB_OK;
    embed_first_kernel<<<cdiv(n, 256), 256, 0, s>>>(ids, first, n, V);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}
// partial[blockIdx.x] = sum of squares of the rows owned by this block's tokens (first occurrences only)
__global__ void embed_rows_sumsq_kernel(const float* __restrict__ dW, const int64_t* __restrict__ ids,
                                        const int* __restrict__ first, int n, int H, int V, float* __restrict__ partial) {
    __shared__ float sh[8];
    float acc = 0.f;
    for (int t = blockIdx.x; t < n; t += gridDim.x) {
        const int64_t id = ids[t];
        if (id < 0 || id >= V || first[id] != t) continue;
        for (int j = threadIdx.x; j < H; j += blockDim.x) {
            float v = dW[id * (int64_t)H + j];
            acc += v * v;
        }
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sh[i];
        partial[blockIdx.x] = t;
    }
}
int embed_rows_sumsq(const float* dW, const int64_t* ids, const int* first, int n, int H, int V, float* partial,
                     int nblocks, cudaStream_t s) {
    embed_rows_sumsq_kernel<<<nblocks, 256, 0, s>>>(dW, ids, first, n, H, V, partial);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}
__global__ void embed_rows_update_kernel(float* __restrict__ W, float* __restrict__ dW, const int64_t* __restrict__ ids,
                                         const int* __restrict__ first, int n, int H, int V, float lr,
                                         const float* __restrict__ scalars, bool write_g) {
    const int t = blockIdx.x;
    const int64_t id = ids[t];
    if (id < 0 || id >= V || first[id] != t) return;
    const float coef = scalars[1];
    for (int j = threadIdx.x; j < H; j += blockDim.x) {
        float g = dW[id * (int64_t)H + j] * coef;
        if (write_g) dW[id * (int64_t)H + j] = g;
        W[id * (int64_t)H + j] -= lr * g;
    }
}
int embed_rows_update(float* W, float* dW, const int64_t* ids, const int* first, int n, int H, int V, float lr,
                      const float* scalars, bool write_g, cudaStream_t s) {
    if (!n) return ZRB_OK;
    embed_rows_update_kernel<<<n, 256, 0, s>>>(W, dW, ids, first, n, H, V, lr, scalars, write_g);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

__global__ void dropout_mask_kernel(MaskSrc m, int64_t n, uint8_t* __restrict__ out) {
    int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (4 * g >= n) return;
    uint32_t bits = m.active ? mask_keep4(m, (uint64_t)g, (uint64_t)n) : 0xFu;
    for (int i = 0; i < 4; ++i)
        if (4 * g + i < n) out[4 * g + i] = (bits >> i) & 1u;
}
int dropout_mask_bytes(MaskSrc m, int64_t n, uint8_t* out, cudaStream_t s) {
    if (!n) return ZRB_OK;
    dropout_mask_kernel<<<cdiv((n + 3) / 4, 256), 256, 0, s>>>(m, n, out);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
