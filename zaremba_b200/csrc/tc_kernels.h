// Launchers used only by the tensor-core engine.
#pragma once
#include "kernels.h"
#include "tc_host.h"

namespace zrb {

constexpr float kGradScale = 1024.f;   // fp16 gradient images hold kGradScale * value (exact power of two)

int convert_pad_f16(const float* src, int64_t ld_src, __half* dst, int64_t ld_dst, int rows, int cols, float scale,
                    cudaStream_t s);
int colsum_h_scratch_floats(int M);
int colsum_h(const __half* A, int64_t ld, float* out, float* out2, int N, int M, float inv_scale, float* scratch,
             cudaStream_t s);

// cell pointwise with fp16 side outputs (tc_cell.cu).  rm: recurrent mask of element b*H + j (variational mode), applied
// to h_raw_h (the next step's operand) forward and to dh_rec backward
int lstm_cell_fwd_tc(float* pre, const float* c_prev, float* c_out, float* h_raw, __half* h_raw_h, __half* y_h,
                     int64_t ld_h, int B, int H, int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s);
int lstm_cell_bwd_tc(const float* dy_post, const float* dh_rec, float* dc, const float* gates, const float* c_t,
                     const float* c_prev, float* dG, __half* dG_h, int64_t ld_g, int B, int H, int64_t elem_off,
                     int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s);

// ---- persistent recurrence (lstm_rec_fwd.cu / lstm_rec_bwd.cu) ---------------------------------------
struct RecPlan {
    int ok;      // shape fits the persistent kernel (else the per-timestep path is used)
    int U;       // hidden units per CTA
    int G;       // 8-row groups of the weight slice (ceil(4U/8))
    int GB;      // 8-row groups of the batch operand (ceil(B/8))
    int Kc;      // 8-element K chunks of the whole contraction
    int nCTA;
    int smem;
    int KS;      // K-split: CTAs that share one set of output rows, each holding 1/KS of the contraction (clusters)
    int KcS;     // K chunks per CTA (Kc / KS)
    int GBi;     // 8-row batch groups of the operand images (GB, or padded so that the MMA's N is a multiple of 16)
};
size_t rec_smem_bytes(int Kc, int G, int GB);
// Where a persistent kernel that gave up on a wait (rec_common.cuh: RecWatch) reports it: `flag` is the device word the
// spinning threads poll, `host` a mapped host word the host reads without synchronising.  Owned by the context.
struct RecWatchdog {
    unsigned int* flag = nullptr;
    unsigned int* host = nullptr;
};
int rec_fwd_plan(int H, int B, RecPlan* plan);
int pack_whh_fwd(const float* W, __half* img, int H, const RecPlan& p, cudaStream_t s);
// h0_img: the B operand of step 0 (image of the state entering the window, built by fwd_prep); h_img slot t+1 is
// written by step t.  The grid-barrier counter is never reset between launches: `counter_base` is its value when
// the launch starts (the caller adds T * nCTA per launch).
int lstm_rec_fwd(const RecPlan& p, const RecWatchdog& wd, const __half* w_img, const __half* h0_img, __half* h_img, float* gates,
                 const float* c0, float* cst, float* h_last, float* c_last, __half* hprev_h, __half* y_h,
                 unsigned int* counter, unsigned int counter_base, int T, int B, int H, int Hp, MaskSrc m, MaskSrc rm,
                 cudaStream_t s, long long* trace = nullptr, float* h_f32 = nullptr);   // h_f32: optional [N,H] fp32 copy of h_t
// m: the output site's mask (period B*H in the variational mode); rm: the recurrent mask of element b*H + j, applied to
// the operand images and hprev_h (never to h_last, h_f32 or the input of m).
// Everything the forward needs from the incoming state and tokens in ONE launch (it replaced 9: five device
// copies, two fp16 conversions, two image packs): h0s/c0s = copies of the incoming (h, c) (the caller may pass
// the same buffers for the outgoing state), hprev_h rows [0,B) = half(h0) with zeroed pad columns, h0_img = the
// UMMA-layout image [kc][g][r][e] = half(h0[b = g*8+r, k = kc*8+e]) (null: not built), x_saved = x.  Variational mode:
// the half(h0) rows and the image hold h0 * rm[l] (element b*H + k); h0s stays unmasked.
struct FwdPrep {
    const float* in_h[ZRB_MAX_LAYERS];
    const float* in_c[ZRB_MAX_LAYERS];
    float* h0s[ZRB_MAX_LAYERS];
    float* c0s[ZRB_MAX_LAYERS];
    __half* hprev_h[ZRB_MAX_LAYERS];
    __half* h0_img[ZRB_MAX_LAYERS];
    MaskSrc rm[ZRB_MAX_LAYERS];
    const int64_t* x;
    int64_t* x_saved;
    int L, B, H, Hp, GB, Kc, N;
};
int fwd_prep(const FwdPrep& a, cudaStream_t s);
// SGD update of one matrix fused with its fp16 image rebuild (optim_tc.cu)
int update_pack(float* p, float* g, int rows, int cols, float lr, const float* scalars, __half* row_img, int64_t ld,
                __half* fwd_img, const RecPlan* fp, __half* bwd_img, const RecPlan* bp, bool write_g, cudaStream_t s,
                bool pdl = false);   // pdl: programmatic dependent of the (forward recurrence) kernel enqueued before it
// the same kernels with the dynamic-evaluation rule (dyneval_elem): theta_g tg and r at p's offsets (r unused under the
// SGD rule, a.rbar null); g is read, never written; the same images
int update_pack_dyn(float* p, float* g, const float* tg, const float* r, int rows, int cols, const DynArgs& a,
                    __half* row_img, int64_t ld, __half* fwd_img, const RecPlan* fp, __half* bwd_img, const RecPlan* bp,
                    cudaStream_t s);
int rec_bwd_plan(int H, int B, RecPlan* plan);   // U = units per CTA, nCTA = 4 * clusters
int pack_whh_bwd(const float* W, __half* img, int H, const RecPlan& p, cudaStream_t s);
int lstm_rec_bwd(const RecPlan& p, const RecWatchdog& wd, const __half* w_img, __half* g_img, const float* dy, const float* gates,
                 const float* cst, const float* c0, __half* dG_h, unsigned int* counter, unsigned int counter_base, int T,
                 int B, int H, int G4p, MaskSrc m, MaskSrc rm, cudaStream_t s, long long* trace = nullptr, float* db1 = nullptr,
                 float* db2 = nullptr,    // db1 / db2: bias gradients sum_{t,b} dG [4H] written by the kernel (or null)
                 unsigned int* resident_flag = nullptr, unsigned int resident_value = 0, float* db_scratch = nullptr);
// resident_flag: CTA 0 stores resident_value there once every CTA of the grid has arrived at the first grid barrier,
// i.e. the whole persistent grid holds its SMs: a stream gated on it (cuStreamWaitValue32) can then start work that
// must only take the SMs this kernel leaves free (the data-parallel bucket all-reduce).

}  // namespace zrb
