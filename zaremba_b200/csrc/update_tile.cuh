// The tile kernels of the fused weight update: each thread updates a tile of 8 rows of one matrix with a rule (SGD,
// dynamic evaluation, SGD + iterate averaging, the average swap, Adam) and writes the fp16 operand images of the new
// weights from registers.  Shared by optim_tc.cu (SgdRule, DynRule), average_tc.cu (AvgRule, SwapRule) and adam_tc.cu
// (AdamRule); every translation unit instantiates the kernels of its own rules.
#pragma once
#include "tc_kernels.h"

namespace zrb {

struct PackSpec {
    __half* row_img;     // [rows, ld] row-major image or null
    int64_t ld;
    __half* fwd_img;     // recurrent forward slices  [cta][kc][g][8][8] or null
    int fU, fG, fKc, fKS;   // units per cluster (KS * U), row groups, K chunks per CTA, K-split factor
    __half* bwd_img;     // recurrent backward slices [cluster][4][kc][g][8][8] or null
    int bUC, bG, bKc, bS;   // units per cluster, row groups, K chunks per CTA, K-split factor per gate
    int write_g;         // store coef * g back into the gradient buffer (clip_grad_norm_'s in-place scaling)
    int pdl;             // launched as a programmatic dependent of the forward recurrence kernel enqueued before it
                         // (deferred update, zrb_set_lazy_update): release the next dependent at once, and block 0 waits
                         // for the primary before it exits so that the grid cannot complete before the primary has
};

__device__ __forceinline__ void pdl_prologue(const PackSpec& sp) {
    if (sp.pdl && threadIdx.x == 0) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_epilogue(const PackSpec& sp) {
    if (sp.pdl && blockIdx.x == 0 && threadIdx.x == 0) asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <int VEC> struct VecT;
template <> struct VecT<4> { using type = float4; };
template <> struct VecT<2> { using type = float2; };
template <> struct VecT<1> { using type = float; };

template <int VEC>
__device__ __forceinline__ void load_vec(const float* p, float (&v)[VEC]) {
    typename VecT<VEC>::type t = __ldcs(reinterpret_cast<const typename VecT<VEC>::type*>(p));
    const float* f = reinterpret_cast<const float*>(&t);
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = f[i];
}
// 8- and 16-byte stores of fp16 images, written out: from a struct assignment the compiler may emit 4-byte stores
// when it cannot prove the alignment of the computed address.  (Nothing in the update kernels reads the images.)
__device__ __forceinline__ void st_v2(__half* dst, uint32_t a, uint32_t b) {
    asm volatile("st.global.v2.b32 [%0], {%1, %2};" ::"l"(dst), "r"(a), "r"(b));
}
__device__ __forceinline__ void st_v4(__half* dst, const uint4& v) {
    asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}

// fp16 image of VEC consecutive values, packed two per word: w[k] = (half(v[2k]), half(v[2k+1])) with the low half
// first, one paired conversion per word (the same bits as __float2half_rn per element); VEC = 1: w[0] = half(v[0])
template <int VEC>
__device__ __forceinline__ void pack_row(const float (&v)[VEC], uint32_t (&w)[(VEC + 1) / 2]) {
    if constexpr (VEC == 1) {
        w[0] = __half_as_ushort(__float2half_rn(v[0]));
    } else {
#pragma unroll
        for (int k = 0; k < VEC / 2; ++k) {
            const __half2 h = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
            w[k] = *reinterpret_cast<const uint32_t*>(&h);
        }
    }
}
// pack_row's words in one store (VEC-element aligned destination)
template <int VEC>
__device__ __forceinline__ void store_halves(__half* dst, const uint32_t (&w)[(VEC + 1) / 2]) {
    if constexpr (VEC == 4) st_v2(dst, w[0], w[1]);
    else if constexpr (VEC == 2) *reinterpret_cast<uint32_t*>(dst) = w[0];
    else *reinterpret_cast<unsigned short*>(dst) = (unsigned short)w[0];
}

template <int VEC>
__device__ __forceinline__ void store_vec(float* p, const float (&v)[VEC]) {
    typename VecT<VEC>::type t;
    float* f = reinterpret_cast<float*>(&t);
#pragma unroll
    for (int i = 0; i < VEC; ++i) f[i] = v[i];
    __stcs(reinterpret_cast<typename VecT<VEC>::type*>(p), t);
}

// Both update kernels give each thread a tile of kTileRows rows x VEC columns and issue every load of the tile (g and
// p, and the rule's own loads) before its first store: (16 B of g + 16 B of p) x 8 rows = 256 B in flight per thread
// at 4 columns under SgdRule (512 B under DynRule<true>), instead of one dependent round trip per row.  ptxas (CUDA
// 12.9) gives the SgdRule 4-column kernels 96 registers (W_hh) and 80 (the others), so an SM holds 5 / 6 blocks of
// 128 threads: 160 / 192 KB of loads in flight per SM.
constexpr int kTileRows = 8;
constexpr int kUpdThreads = 128;

// A rule is init(), apply(off, p row, g row) (the new p, and g as the kernel may store it), and three hooks for
// streams of its own that the kernel stores (iterate averaging, Adam's moments): load(off, e, tile) with the tile's
// loads, finish(e, p row, g row, tile) after apply (it may still change p and g: Adam's update needs the tile),
// store(off, e, tile) after the tile's p / g stores.  A rule without such a stream derives from NoTileRule.
struct NoTileRule {
    template <int VEC> struct Tile {};
    template <int VEC> __device__ __forceinline__ void load(int64_t, int, Tile<VEC>&) const {}
    template <int VEC> __device__ __forceinline__ void finish(int, float (&)[VEC], float (&)[VEC], Tile<VEC>&) const {}
    template <int VEC> __device__ __forceinline__ void store(int64_t, int, const Tile<VEC>&) const {}
};

// SgdRule: g *= coef (clip_grad_norm_, coef = scalars[1]); p -= lr*g, with g stored back when PackSpec::write_g asks
struct SgdRule : NoTileRule {
    float lr;
    const float* scalars;
    float coef;
    static constexpr bool kMayWriteG = true;
    static constexpr int kWhhMinBlocks = 5;   // W_hh kernel: 5 blocks of 128 per SM (at most 102 registers)
    __device__ __forceinline__ void init() { coef = scalars[1]; }
    template <int VEC>
    __device__ __forceinline__ void apply(int64_t, float (&pv)[VEC], float (&gv)[VEC]) const {
#pragma unroll
        for (int x = 0; x < VEC; ++x) { gv[x] *= coef; pv[x] = sgd_elem(pv[x], gv[x], lr); }
    }
};

// load rows e < n (at off + e * stride) of g and p (and the rule's tile), then apply the rule to each; nothing is
// stored here
template <int VEC, class Rule>
__device__ __forceinline__ void tile_update(const float* __restrict__ p, const float* __restrict__ g, int64_t off,
                                            int stride, int n, const Rule& rule, float (&pv)[kTileRows][VEC],
                                            float (&gv)[kTileRows][VEC], typename Rule::template Tile<VEC>& tile) {
#pragma unroll
    for (int e = 0; e < kTileRows; ++e) {
        if (e < n) {
            load_vec<VEC>(g + off + (int64_t)e * stride, gv[e]);
            load_vec<VEC>(p + off + (int64_t)e * stride, pv[e]);
            rule.template load<VEC>(off + (int64_t)e * stride, e, tile);
        }
    }
#pragma unroll
    for (int e = 0; e < kTileRows; ++e) {
        if (e < n) {
            rule.template apply<VEC>(off + (int64_t)e * stride, pv[e], gv[e]);
            rule.template finish<VEC>(e, pv[e], gv[e], tile);
        }
    }
}

template <int VEC, class Rule>
__device__ __forceinline__ void tile_store(float* __restrict__ p, float* __restrict__ g, int64_t off, int stride, int n,
                                           bool write_g, const float (&pv)[kTileRows][VEC],
                                           const float (&gv)[kTileRows][VEC], const Rule& rule,
                                           const typename Rule::template Tile<VEC>& tile) {
#pragma unroll
    for (int e = 0; e < kTileRows; ++e) {
        if (e < n) {
            if (write_g) store_vec<VEC>(g + off + (int64_t)e * stride, gv[e]);
            store_vec<VEC>(p + off + (int64_t)e * stride, pv[e]);
            rule.template store<VEC>(off + (int64_t)e * stride, e, tile);
        }
    }
}

// The grid is 1-D and row-major over the tiles: block b = (row group) * col_tiles + (column tile), decoded once per
// block.  The blocks resident at one time then cover a band of whole rows, so the kernel streams through the matrix
// like a flat copy, and the 32-byte sectors shared by two column tiles (rows are only 16-byte aligned when cols % 8
// == 4) are read by two blocks that run at about the same time.

// matrix [rows, cols] (cols % VEC == 0): the rule's update of p; row-major fp16 image of the new p.  Block b: rows
// 8r..8r+7 and, for thread t, columns (ct * blockDim.x + t) * VEC + 0..VEC-1, where (r, ct) = divmod(b, col_tiles).
template <int VEC, class Rule>
__global__ void __launch_bounds__(kUpdThreads) update_pack_kernel(float* __restrict__ p, float* __restrict__ g, int rows,
                                                                  int cols, int col_tiles, Rule rule, PackSpec sp) {
    pdl_prologue(sp);
    rule.init();
    const unsigned rg = blockIdx.x / (unsigned)col_tiles, ct = blockIdx.x - rg * col_tiles;
    const int c = (ct * blockDim.x + threadIdx.x) * VEC;
    const int r0 = rg * kTileRows, n = min(kTileRows, rows - r0);
    if (c < cols) {
        const int64_t off = (int64_t)r0 * cols + c;
        float pv[kTileRows][VEC], gv[kTileRows][VEC];
        typename Rule::template Tile<VEC> tile;
        tile_update<VEC>(p, g, off, cols, n, rule, pv, gv, tile);
        tile_store<VEC>(p, g, off, cols, n, Rule::kMayWriteG && sp.write_g, pv, gv, rule, tile);
        if (sp.row_img) {
#pragma unroll
            for (int e = 0; e < kTileRows; ++e) {
                if (e < n) {
                    uint32_t w[(VEC + 1) / 2];
                    pack_row<VEC>(pv[e], w);
                    store_halves<VEC>(sp.row_img + (int64_t)(r0 + e) * sp.ld + c, w);
                }
            }
        }
    }
    pdl_epilogue(sp);
}

// W_hh [4H, H] with both recurrent images.  Block b owns rows j0..j0+7 (j0 = 8 * (b / col_tiles)) of all four gate
// blocks and 8 * VEC columns per warp (column tile b % col_tiles); lane l of a warp holds gate q = l & 3 and columns c..c+VEC-1, c = (the warp's first column)
// + (l >> 2) * VEC.  With the four gates of a unit on adjacent lanes, rows 4u..4u+3 of a forward-slice 8x8 block (one
// K chunk) are written by one instruction: 64 contiguous bytes.  The backward image's 16-byte vectors hold 8
// consecutive K indices (= rows j0..j0+7) of one unit (= column), so a thread's column tile gives them whole.
template <int VEC, class Rule>
__global__ void __launch_bounds__(kUpdThreads, Rule::kWhhMinBlocks) update_pack_whh_kernel(float* __restrict__ p, float* __restrict__ g,
                                                                      int H, int col_tiles, Rule rule, PackSpec sp) {
    pdl_prologue(sp);
    rule.init();
    const int lane = threadIdx.x & 31, q = lane & 3;
    const unsigned jb = blockIdx.x / (unsigned)col_tiles, ct = blockIdx.x - jb * col_tiles;
    const int c = ((ct * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 8 + (lane >> 2)) * VEC;
    const int j0 = jb * kTileRows, n = min(kTileRows, H - j0);
    uint32_t hw[kTileRows][(VEC + 1) / 2];   // pack_row of each row; 0 (= half(0)) for rows past H and dead lanes
    if (c < H) {
        const int64_t off = ((int64_t)q * H + j0) * H + c;
        float pv[kTileRows][VEC], gv[kTileRows][VEC];
        typename Rule::template Tile<VEC> tile;
        tile_update<VEC>(p, g, off, H, n, rule, pv, gv, tile);
#pragma unroll
        for (int e = 0; e < kTileRows; ++e) {
            if (e < n) {
                pack_row<VEC>(pv[e], hw[e]);
            } else {
#pragma unroll
                for (int k = 0; k < (VEC + 1) / 2; ++k) hw[e][k] = 0;
            }
        }
        tile_store<VEC>(p, g, off, H, n, Rule::kMayWriteG && sp.write_g, pv, gv, rule, tile);
        if (sp.row_img) {
#pragma unroll
            for (int e = 0; e < kTileRows; ++e)
                if (e < n) store_halves<VEC>(sp.row_img + (int64_t)(q * H + j0 + e) * sp.ld + c, hw[e]);
        }
        if (sp.fwd_img) {   // slice of the CTA owning unit j, row 4u+q; K indices c..c+VEC-1 share a K chunk
            const unsigned kc = (unsigned)c >> 3, kq = kc / (unsigned)sp.fKc, kcl = kc - kq * sp.fKc;
            unsigned cluster = (unsigned)j0 / (unsigned)sp.fU, u = j0 - cluster * sp.fU;
#pragma unroll
            for (int e = 0; e < kTileRows; ++e) {
                if (e < n) {
                    const unsigned row = 4 * u + q, cta = cluster * sp.fKS + kq;
                    store_halves<VEC>(sp.fwd_img + ((int64_t)(cta * sp.fKc + kcl) * sp.fG + (row >> 3)) * 64 +
                                          (row & 7) * 8 + (c & 7), hw[e]);
                }
                if (++u == (unsigned)sp.fU) { u = 0; ++cluster; }
            }
        }
    } else {
#pragma unroll
        for (int e = 0; e < kTileRows; ++e)
#pragma unroll
            for (int k = 0; k < (VEC + 1) / 2; ++k) hw[e][k] = 0;
    }
    if (sp.bwd_img) {   // units c..c+VEC-1, rank q, K chunk jb: one 16-byte vector per unit
        // column x's vector: (half(row 2m, x), half(row 2m + 1, x)) for m = 0..3, taken out of the row words
        uint4 v[VEC];
#pragma unroll
        for (int x = 0; x < VEC; ++x) {
            uint32_t w[4];
#pragma unroll
            for (int m = 0; m < 4; ++m)
                w[m] = VEC == 1 ? hw[2 * m][0] | (hw[2 * m + 1][0] << 16)
                                : __byte_perm(hw[2 * m][x >> 1], hw[2 * m + 1][x >> 1], (x & 1) ? 0x7632 : 0x5410);
            v[x] = make_uint4(w[0], w[1], w[2], w[3]);
        }
        const unsigned rank = q * sp.bS + jb / (unsigned)sp.bKc, kcl = jb - (jb / sp.bKc) * sp.bKc;
        __half* base = sp.bwd_img + (int64_t)kcl * sp.bG * 64;
        auto put = [&](int unit, const uint4& val) {
            if (unit < H) {
                const unsigned cl = (unsigned)unit / (unsigned)sp.bUC, u = unit - cl * sp.bUC;
                st_v4(base + (int64_t)((cl * 4 * sp.bS + rank) * sp.bKc) * sp.bG * 64 + (u >> 3) * 64 + (u & 7) * 8, val);
            }
        };
        if constexpr (VEC == 1) {
            put(c, v[0]);   // lanes l and l + 4 hold adjacent units: whole sectors already
        } else {
            // lanes l and l ^ 4 hold units a..a+2*VEC-1 between them; after a swap of half their vectors, store i writes
            // unit a+2i from the lower lane and a+2i+1 from the upper one, the two halves of one 32-byte sector
            const bool lower = ((lane >> 2) & 1) == 0;
            const int a = lower ? c : c - VEC;
            uint4 recv[VEC / 2];
#pragma unroll
            for (int m = 0; m < VEC / 2; ++m) {
                const uint4 s = lower ? v[2 * m + 1] : v[2 * m];
                recv[m] = make_uint4(__shfl_xor_sync(0xffffffffu, s.x, 4), __shfl_xor_sync(0xffffffffu, s.y, 4),
                                     __shfl_xor_sync(0xffffffffu, s.z, 4), __shfl_xor_sync(0xffffffffu, s.w, 4));
            }
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                if (lower) put(a + 2 * i, i < VEC / 2 ? v[2 * i] : recv[i - VEC / 2]);
                else put(a + 2 * i + 1, i < VEC / 2 ? recv[i] : v[2 * (i - VEC / 2) + 1]);
            }
        }
    }
    pdl_epilogue(sp);
}

template <int VEC, class Rule>
static int update_pack_launch(float* p, float* g, int rows, int cols, const Rule& rule, const PackSpec& sp, bool whh,
                              int pdl_smem, cudaStream_t s) {
    // one tile per thread, the grid sized to the tiles: W_hh 8 rows of the 4 gates x 8 * VEC columns per warp, other
    // matrices 8 rows x VEC columns per thread (narrower blocks when the matrix is narrow)
    const int cv = cols / VEC;
    int threads = kUpdThreads, col_tiles;
    if (whh) {
        col_tiles = (cv + 8 * (threads / 32) - 1) / (8 * (threads / 32));
    } else {
        threads = min(kUpdThreads, (cv + 31) / 32 * 32);
        col_tiles = (cv + threads - 1) / threads;
    }
    const dim3 grid((unsigned)(((rows / (whh ? 4 : 1)) + kTileRows - 1) / kTileRows * col_tiles));
    if (pdl_smem > 0) {
        // beside the persistent forward recurrence: pdl_smem is more dynamic shared memory than that kernel leaves free
        // on its SMs (rec_beside_smem), which keeps these blocks on the SMs it does not occupy, off the latency-critical
        // ones
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = grid; cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = (size_t)pdl_smem; cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        if (whh) {
            ZRB_CUDA(cudaFuncSetAttribute(update_pack_whh_kernel<VEC, Rule>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          pdl_smem));
            ZRB_CUDA(cudaLaunchKernelEx(&cfg, update_pack_whh_kernel<VEC, Rule>, p, g, cols, col_tiles, rule, sp));
        } else {
            ZRB_CUDA(cudaFuncSetAttribute(update_pack_kernel<VEC, Rule>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          pdl_smem));
            ZRB_CUDA(cudaLaunchKernelEx(&cfg, update_pack_kernel<VEC, Rule>, p, g, rows, cols, col_tiles, rule, sp));
        }
        count_launch();
        return ZRB_OK;
    }
    if (whh) update_pack_whh_kernel<VEC, Rule><<<grid, threads, 0, s>>>(p, g, cols, col_tiles, rule, sp);
    else update_pack_kernel<VEC, Rule><<<grid, threads, 0, s>>>(p, g, rows, cols, col_tiles, rule, sp);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// align: OR of every pointer the rule streams besides p and g (their alignment picks the access width too)
template <class Rule>
static int update_pack_rule(float* p, float* g, int rows, int cols, const Rule& rule, uintptr_t align,
                            const WeightImages& img, bool write_g, cudaStream_t s, int pdl_smem) {
    const RecPlan *fp = img.fplan, *bp = img.bplan;
    PackSpec sp;
    sp.write_g = write_g ? 1 : 0;
    sp.pdl = pdl_smem > 0 ? 1 : 0;
    sp.row_img = img.row; sp.ld = img.ld;
    sp.fwd_img = img.fwd; sp.fKS = fp ? fp->KS : 1; sp.fU = fp ? fp->KS * fp->U : 1; sp.fG = fp ? fp->G : 1;
    sp.fKc = fp ? fp->KcS : 1;
    sp.bwd_img = img.bwd; sp.bS = bp ? bp->KS : 1; sp.bUC = bp ? 4 * bp->KS * bp->U : 4; sp.bG = bp ? bp->G : 1;
    sp.bKc = bp ? bp->KcS : 1;
    const bool whh = (img.fwd || img.bwd) && rows == 4 * cols;
    const uintptr_t all = ((uintptr_t)p) | ((uintptr_t)g) | align;
    const bool al16 = (all & 15) == 0, al8 = (all & 7) == 0;
    if (cols % 4 == 0 && al16) return update_pack_launch<4>(p, g, rows, cols, rule, sp, whh, pdl_smem, s);
    if (cols % 2 == 0 && al8) return update_pack_launch<2>(p, g, rows, cols, rule, sp, whh, pdl_smem, s);
    return update_pack_launch<1>(p, g, rows, cols, rule, sp, whh, pdl_smem, s);
}

}  // namespace zrb
