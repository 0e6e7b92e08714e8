// Helpers shared by the persistent recurrence kernels (forward / backward).
#pragma once
#include <string.h>
#include "tc_common.cuh"
#include "tc_kernels.h"

namespace zrb {
using namespace tc;

constexpr int kRecEpiWarps = 8;                       // warps 0-7: cell math
constexpr int kRecEpiThreads = kRecEpiWarps * 32;
constexpr int kRecMmaWarp = 8;                        // warps 8..11: one warpgroup issues the step's wgmma chain and hands the
constexpr int kRecMmaWarps = 4;                       //   accumulators (registers) to their readers
constexpr int kRecMmaThreads = kRecMmaWarps * 32;
constexpr int kRecLoadWarp = kRecMmaWarp + kRecMmaWarps;   // lane 0: grid-barrier wait + bulk copies
constexpr int kRecThreads = (kRecLoadWarp + 1) * 32;
constexpr int kRecPieces = 4;                         // operand image arrives in this many bulk copies, so that the MMAs
                                                      // start when the first quarter of K has landed
constexpr int kRecMaxCell = 2;                        // (unit, batch) cells per epilogue thread
// The K-split plans' first choice of U (rec_fwd_plan / rec_bwd_plan): each of the 256 epilogue threads owns at most one
// (unit, batch) cell, and the grid of nCTA leaves at least an eighth of the SMs to the kernels launched beside it (the
// deferred weight update, the weight gradients).  When no U meets both, the plans take the largest U that fits: two
// cells for some threads cost less than a grid that leaves the work beside it a handful of SMs (DESIGN.md section 4.1)
inline bool rec_split_first_choice(int U, int B, int nCTA, int nsm) {
    return U * B <= kRecEpiThreads && nCTA <= nsm - nsm / 8;
}
// ---- watchdog -------------------------------------------------------------------------------------
// Every wait of the persistent kernels is bounded.  A wait that runs out (a lost wake-up, a grid that is not co-resident)
// publishes a code in the context's abort word; from then on EVERY wait of EVERY thread returns at once (a thread that
// has seen the word set stops waiting for good), so the kernel runs to its end through its unchanged barrier skeleton --
// producing garbage, but terminating, with the CUDA context intact.  The host finds the code in a mapped host word at its
// next API call and fails the zrb context (api.cu: watchdog_check).  Nothing on the fast path but a register test.
// host: the kernel argument for one launch (ZRB_SPIN_CYCLES shortens the time-out; read once), and the fault injection
// of tests/test_gpu_watchdog.py: ZRB_FAULT_BARRIER_BASE="fwd" / "bwd" makes that kernel's launches expect one arrival
// more than the grid will ever deliver -- every CTA then sits at its first grid barrier like after a lost wake-up.
static inline RecWatch rec_watch_args(const RecWatchdog& wd) {
    static const long long spin = [] { const char* e = getenv("ZRB_SPIN_CYCLES"); long long v = e ? atoll(e) : 0; return v > 0 ? v : 6000000000ll; }();
    RecWatch w;
    w.flag = wd.flag; w.host = wd.host; w.spin_cycles = spin;
    return w;
}
static inline unsigned int rec_fault_base(const char* which) {
    static const char* fault = getenv("ZRB_FAULT_BARRIER_BASE");
    return (fault && !strcmp(fault, which)) ? 1u : 0u;
}
enum { kWaitWeights = 1, kWaitOperand = 2, kWaitAcc = 3, kWaitRecv = 4, kWaitGrid = 5 };

__device__ __forceinline__ unsigned int ld_relaxed_gpu(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// code = wait kind | CTA << 8 | step << 20
static __device__ __noinline__ void rec_give_up(unsigned int* flag, unsigned int* host, int kind, int step) {
    const unsigned int code = (unsigned int)kind | ((unsigned int)(blockIdx.x & 0xFFF) << 8) | ((unsigned int)(step & 0xFFF) << 20);
    if (atomicCAS(flag, 0u, code) == 0u) {
        asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(host), "r"(code) : "memory");
        __threadfence_system();
    }
}
// one slow-path visit of a spinning thread (every few thousand polls): true = stop waiting (for good), because the word
// is set or because this wait ran out -- the caller then reports it with rec_give_up (a no-op once the word is set)
__device__ __forceinline__ bool rec_spin_expired(const RecWatch& w, long long& t0) {
    if (ld_relaxed_gpu(w.flag) != 0u) return true;
    const long long now = clock64();
    if (t0 == 0) { t0 = now; return false; }
    return now - t0 > w.spin_cycles;
}
__device__ __forceinline__ bool rec_spin_check(const RecWatch& w, long long& t0, int kind, int step) {
    if (!rec_spin_expired(w, t0)) return false;
    rec_give_up(w.flag, w.host, kind, step);
    return true;
}

__device__ __forceinline__ void bounded_mbar_wait(uint64_t* bar, uint32_t parity, const RecWatch& w, bool& dead, int kind,
                                                  int step) {
    if (dead) return;
    uint32_t n = 0;
    long long t0 = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++n & 0xFFFu) == 0 && rec_spin_check(w, t0, kind, step)) { dead = true; return; }
    }
}

__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}


// ---- the MMA warpgroup ----------------------------------------------------------------------------
// True on every MMA thread when any of them has `v` set (named barrier 2 over the warpgroup): a wait that gave up on one
// thread must stop all four warps, since each wgmma needs the whole warpgroup.
__device__ __forceinline__ bool rec_mma_any(bool v) {
    uint32_t r;
    asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 q, %1, 0;\n\tbar.red.or.pred p, 2, %2, q;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(r)
                 : "r"((uint32_t)v), "n"(kRecMmaThreads)
                 : "memory");
    return r != 0;
}

// The accumulator row that register pair (mt, h) of MMA thread t (0..127) holds: each thread holds four rows at most,
// so a kernel works out where each of them goes once, before its step loop (tc_common.cuh: wgmma_row).
__device__ __forceinline__ int rec_acc_row(int t, int mt, int h) { return 64 * mt + wgmma_row(t, h); }

// bounded_mbar_wait for the span where wgmmas are in flight: no call, no write to `dead`.  false = this thread stopped
// waiting; the caller reports it with rec_give_up once nothing is in flight.
__device__ __forceinline__ bool rec_chain_wait(uint64_t* bar, uint32_t parity, const RecWatch& w) {
    uint32_t n = 0;
    long long t0 = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++n & 0xFFFu) == 0 && rec_spin_expired(w, t0)) return false;
    }
    return true;
}

// One step of the MMA warpgroup: D[64 MT x 8 NB] = A[64 MT rows x K] * B[8 NB x K]^T, K in ksteps steps of 16 that arrive
// in kRecPieces pieces (bar_b[pc], phase `parity`).  Both operands are K-major in the canonical no-swizzle layout: 8x8
// core matrices of 128 B, 8-row groups 128 B apart, the two K halves of a step lbo bytes apart.  Then emit(mt, h, col,
// v0, v1) for every accumulator pair (row rec_acc_row(t, mt, h), columns col, col + 1).  Returns with `dead` set (on
// every MMA thread) when a wait gave up.
//
// The whole step is ONE asynchronous chain: the wgmmas go out back to back, and the only wait for them is the
// wgmma_wait<0> before the accumulators are read.  ptxas serialises every wgmma (a wait after each) when it finds a
// call or a branch it cannot prove warp-uniform between them while accumulators are live, so inside the chain: the
// operand waits call nothing (rec_chain_wait), the warpgroup's vote is the only thing that decides whether the chain
// goes on, and a warpgroup that gives up issues no further wgmma by running the remaining pieces with zero K steps
// rather than by leaving the loop.  Everything that depends on one thread (the trace stamp, rec_give_up) is outside.
template <int NB, int MT, class Emit>
__device__ __forceinline__ void rec_mma_step_nb(uint32_t a_addr, uint32_t b_addr, uint32_t lbo_a, uint32_t lbo_b, int ksteps,
                                                int piece_steps, uint64_t* bar_b, uint32_t parity, const RecWatch& w,
                                                bool& dead, int step, long long* stamp, Emit& emit) {
    constexpr int R = NB * 4;
    float d[MT][R];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int i = 0; i < R; ++i) d[mt][i] = 0.f;
    const int t = (int)threadIdx.x - kRecMmaWarp * 32;
    bool lost = dead ? false : !rec_chain_wait(&bar_b[0], parity, w);
    dead = rec_mma_any(dead || lost);
    if (stamp && t == 0) *stamp = clock64();   // MMA start: the first piece has landed, nothing is in flight yet
    wgmma_fence();
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) wgmma_fence_acc(d[mt]);
    for (int pc = 0; pc < kRecPieces; ++pc) {
        if (pc > 0) {
            if (!dead) lost = !rec_chain_wait(&bar_b[pc], parity, w);
            dead = rec_mma_any(dead || lost);
        }
        const int k0 = pc * piece_steps, k1 = dead ? k0 : min(ksteps, k0 + piece_steps);
        for (int ks = k0; ks < k1; ++ks) {
            const uint64_t db = make_smem_desc(b_addr + ks * 2 * lbo_b, lbo_b, 128, kSwizzleNone);
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {   // rows 64 mt.. start 8 row groups further
                const uint64_t da = make_smem_desc(a_addr + ks * 2 * lbo_a + mt * 1024, lbo_a, 128, kSwizzleNone);
                Wgmma<NB * 8, 0, 0>::mma(d[mt], da, db, 1u);
            }
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) wgmma_fence_acc(d[mt]);
    if (lost) rec_give_up(w.flag, w.host, kWaitOperand, step);
    if (dead) return;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int c8 = 0; c8 < NB; ++c8)
#pragma unroll
            for (int h = 0; h < 2; ++h)
                emit(mt, h, wgmma_col(t, c8), d[mt][4 * c8 + 2 * h], d[mt][4 * c8 + 2 * h + 1]);
}

// the same with N = 8 nb (nb = 1..4: batch up to 32) and MT = mt 64-row tiles (1 or 2) chosen at run time.  Inlined, so
// that the kernel's arguments and `dead` stay in registers and the chain's bounds are known to be warp-uniform.
template <class Emit>
__device__ __forceinline__ void rec_mma_step(int nb, int mt, uint32_t a_addr, uint32_t b_addr, uint32_t lbo_a, uint32_t lbo_b,
                                             int ksteps, int piece_steps, uint64_t* bar_b, uint32_t parity, const RecWatch& w,
                                             bool& dead, int step, long long* stamp, Emit& emit) {
#define ZRB_REC_MMA(NB, MT) \
    rec_mma_step_nb<NB, MT>(a_addr, b_addr, lbo_a, lbo_b, ksteps, piece_steps, bar_b, parity, w, dead, step, stamp, emit)
    switch (nb + 4 * (mt - 1)) {
    case 1: ZRB_REC_MMA(1, 1); break;
    case 2: ZRB_REC_MMA(2, 1); break;
    case 3: ZRB_REC_MMA(3, 1); break;
    case 4: ZRB_REC_MMA(4, 1); break;
    case 5: ZRB_REC_MMA(1, 2); break;
    case 6: ZRB_REC_MMA(2, 2); break;
    case 7: ZRB_REC_MMA(3, 2); break;
    default: ZRB_REC_MMA(4, 2); break;
    }
#undef ZRB_REC_MMA
}

// ---- the cell-math warps ----------------------------------------------------------------------------
// Cell k of cell-math thread tid is cell = tid + kRecEpiThreads * k = b * U + u (u fastest: contiguous j); it exists when
// cell < cells = U * B and u < nu (the CTA's last units may lie past H).  The kernels divide out b = cell / U once,
// before their step loops (cb[k]); the unit then costs one multiply-add per use.
struct RecCell { int b, u; bool ok; };
__device__ __forceinline__ RecCell rec_cell(int tid, int k, int cb_k, int U, int cells, int nu) {
    const int cell = tid + kRecEpiThreads * k, u = cell - cb_k * U;
    return {cb_k, u, cell < cells && u < nu};
}

// 8 bytes into a peer CTA's shared memory; the bytes are counted on that CTA's mbarrier (complete_tx), so the reader
// needs no fence: observing the phase completion makes them visible
__device__ __forceinline__ void st_async_v2(uint32_t cluster_addr, float a, float b, uint32_t cluster_bar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
                 ::"r"(cluster_addr), "f"(a), "f"(b), "r"(cluster_bar) : "memory");
}

// Programmatic dependent launch: once EVERY CTA of this grid has executed this (i.e. the whole persistent grid is
// resident), a kernel enqueued behind it with the programmatic-serialization attribute may start on the SMs this grid
// leaves idle.  Kernels launched normally behind it are unaffected.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// The other side: when THIS kernel was launched with the programmatic-serialization attribute behind a kernel that
// triggers early (the tensor-core GEMMs do), its CTAs become resident -- mbarriers, the resident weight slice on
// its way -- while that kernel is still running; every thread that reads global memory the predecessor wrote calls this
// first.  Returns at once in a normal launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Profiling only (ZRB_REC_TRACE): the 8 launch slots in front of the per-step stamps.  Called by thread 0 of EVERY CTA at
// kernel entry (exit = false) and as its last instruction (exit = true):
//   [0]/[1] CTA 0's clock64 at entry / exit      [2]/[3] CTA 0's %globaltimer (ns) at entry / exit
//   [4] max over CTAs of -(entry %globaltimer)   [5] max over CTAs of the exit %globaltimer   (the host presets both
//   to the most negative value before each launch) -> [5] + [4] = lifetime of the whole grid in ns
__device__ __forceinline__ void rec_launch_stamps(long long* slots, bool cta0, bool exit) {
    long long gt;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    if (cta0) { slots[exit ? 1 : 0] = clock64(); slots[exit ? 3 : 2] = gt; }
    atomicMax(slots + (exit ? 5 : 4), exit ? gt : -gt);
}

// Publish this CTA's global writes of the step and arrive on the grid barrier: one release-RED at gpu scope
// (the bar.sync before it made the other epilogue threads' writes visible to this thread; release is
// cumulative).  The consumers' TMA reads are ordered by THEIR acquire + fence.proxy.async.
__device__ __forceinline__ void grid_counter_arrive(unsigned int* counter) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
}

// spin on a global counter (grid barrier): relaxed polls (a plain L2 round trip each; ld.acquire would add an L1
// invalidate per poll), one acquire fence after the last arrival was seen; bounded like the mbarrier waits
__device__ __forceinline__ void grid_counter_wait(const unsigned int* counter, unsigned int target, const RecWatch& w,
                                                  bool& dead, int step) {
    if (dead) return;
    uint32_t n = 0;
    long long t0 = 0;
    while (ld_relaxed_gpu(counter) < target) {
        if ((++n & 0x3FFu) == 0 && rec_spin_check(w, t0, kWaitGrid, step)) { dead = true; return; }
    }
    asm volatile("fence.acquire.gpu;" ::: "memory");
}

}  // namespace zrb
