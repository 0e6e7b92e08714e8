// The zoneout instantiations of the persistent recurrence kernels (DESIGN.md section 20).  They live in a source of their
// own, so that lstm_rec_fwd.cu and lstm_rec_bwd.cu keep exactly the instantiations they had before the mode existed.
#include "lstm_rec_bwd.cuh"
#include "lstm_rec_fwd.cuh"

namespace zrb {

// The plan functions raise the dynamic shared-memory limit of the mode-off kernels they query, on every device; these
// kernels get it here, once per device (function attributes belong to the device's context).  Null when it fails.
static const void* rec_zoneout_ready(const void* const (&k)[2], int i, bool (&done)[64]) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
    dev &= 63;
    if (!done[dev]) {
        for (const void* f : k)
            if (cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess) {
                set_error("zoneout recurrence kernel: raising its shared-memory limit failed: %s",
                          cudaGetErrorString(cudaGetLastError()));
                return nullptr;
            }
        done[dev] = true;
    }
    return k[i];
}

const void* rec_fwd_zoneout_kernel(bool split) {
    static const void* const k[2] = {(const void*)lstm_rec_fwd_kernel<false, true>,
                                     (const void*)lstm_rec_fwd_kernel<true, true>};
    static bool done[64] = {};
    return rec_zoneout_ready(k, split ? 1 : 0, done);
}

const void* rec_bwd_zoneout_kernel(int S) {
    static const void* const k[2] = {(const void*)lstm_rec_bwd_kernel<1, true>,
                                     (const void*)lstm_rec_bwd_kernel<2, true>};
    static bool done[64] = {};
    return rec_zoneout_ready(k, S == 2 ? 1 : 0, done);
}

}  // namespace zrb
