// Weight update -- the train step's SGD, or dynamic evaluation's rule -- fused with the rebuild of the fp16 operand
// images (tensor-core engine).
// The update pass already holds every new weight in registers; writing its fp16 images from there
// removes the separate pack pass (which re-read 348 MB of fp32 weights per step at the Large config).
#include "update_tile.cuh"

namespace zrb {

// DynRule: the dynamic-evaluation update (dyneval_elem), which also reads theta_g and r at the element's offset and
// never stores g.  (SgdRule and the kernels: update_tile.cuh.)
template <bool RMS>
struct DynRule : NoTileRule {
    const float* tg;     // theta_g, same layout as p
    const float* r;      // RMS statistic, same layout as p (RMS rule only)
    DynArgs a;
    float rbar;
    static constexpr bool kMayWriteG = false;
    // W_hh kernel: at most 128 registers.  Unbounded, ptxas spills a value across the calls of the fp32 division's
    // slow path in the 2-column RMS instantiation.
    static constexpr int kWhhMinBlocks = 4;
    __device__ __forceinline__ void init() { rbar = RMS ? *a.rbar : 0.f; }
    template <int VEC>
    __device__ __forceinline__ void apply(int64_t off, float (&pv)[VEC], float (&gv)[VEC]) const {
        float tv[VEC], rv[VEC];
        load_vec<VEC>(tg + off, tv);
        if constexpr (RMS) load_vec<VEC>(r + off, rv);
#pragma unroll
        for (int x = 0; x < VEC; ++x)
            pv[x] = dyneval_elem<RMS>(pv[x], gv[x], tv[x], RMS ? rv[x] : 0.f, a.lr, a.lam, a.eps, rbar);
    }
};

int update_pack(float* p, float* g, int rows, int cols, float lr, const float* scalars, const WeightImages& img,
                bool write_g, cudaStream_t s, int pdl_smem) {
    SgdRule rule;
    rule.lr = lr; rule.scalars = scalars; rule.coef = 0.f;
    return update_pack_rule(p, g, rows, cols, rule, 0, img, write_g, s, pdl_smem);
}

int update_pack_dyn(float* p, float* g, const float* tg, const float* r, int rows, int cols, const DynArgs& a,
                    const WeightImages& img, cudaStream_t s) {
    const uintptr_t align = ((uintptr_t)tg) | ((uintptr_t)r);
    if (a.rbar) {
        DynRule<true> rule{{}, tg, r, a, 0.f};
        return update_pack_rule(p, g, rows, cols, rule, align, img, false, s, false);
    }
    DynRule<false> rule{{}, tg, nullptr, a, 0.f};
    return update_pack_rule(p, g, rows, cols, rule, align, img, false, s, false);
}

}  // namespace zrb
