// ualm_mailbox.h -- the result mailbox of a submitted batch (ualm_poll_batch), shared by the parity path (ualm_api.cu) and the
// throughput engine (ualm_tp.cu).  Only this header knows its layout.
//
// One mailbox per lane, in pinned host memory mapped into the device's address space (cudaHostAllocMapped), grown only, released
// with the lane.  For a batch of B problems it holds, back to back:
//     B result records | the packed c_xy of the batch | the packed c_yaw of the batch | B int32 ready flags
// (c_xy / c_yaw in problem order, the layout ualm_wait_batch writes).  Ordering: the device writes a problem's record and
// coefficients, then __threadfence_system(), then sets its flag; the host reads a flag with an acquire load and copies the problem
// out only after that.  The device never reads the mailbox (a mapped word read over PCIe inside the solve costs time at every
// read); the host clears the flags at submit, while the lane holds no running batch.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cstring>
#include <vector>

#include "ualm.h"

namespace ualm_mbox {

// where the device writes problem b: res[b], c_xy / c_yaw at the problem's packed offsets, then flag[b] = 1.  flag == nullptr:
// the launch publishes nothing (every launch not made by ualm_submit_batch*)
struct Ptrs {
    ualm_result_t *res;
    double *c_xy, *c_yaw;
    int32_t *flag;
};

#ifdef __CUDACC__
// after the calling warp (all 32 lanes) has written problem b's record and coefficients through `p`: make them visible to the host,
// then raise the flag.  Every lane fences its own writes; lane 0 fences again after the barrier, so the flag store is ordered
// after what the other lanes wrote as well
__device__ __forceinline__ void raise_flag_warp(const Ptrs &p, int b, int lane)
{
    __threadfence_system();
    __syncwarp();
    if (lane == 0) {
        __threadfence_system();
        *(volatile int32_t *)(p.flag + b) = 1;
    }
}
#endif

class Mailbox {
public:
    // Lays the mailbox out for a batch (B problems, piece counts N / M), clears the flags and the per-ticket returned mask, and
    // publishes the problems the device will not solve (skip[b] != 0: over the compiled limits) at once: a zero record with
    // ret_code UALM_ELIMIT and zero coefficients, what ualm_wait_batch returns for them.  Call only while no kernel of the lane runs.
    cudaError_t begin(int B, const int32_t *N, const int32_t *M, const unsigned char *skip)
    {
        B_ = B;
        ocx_.assign(B + 1, 0); ocy_.assign(B + 1, 0);
        for (int b = 0; b < B; b++) { ocx_[b + 1] = ocx_[b] + 12LL * N[b]; ocy_[b + 1] = ocy_[b] + 6LL * M[b]; }
        returned_.assign(B, 0);
        n_returned_ = 0;
        if (B == 0) { host_ = dev_ = Ptrs{}; return cudaSuccess; }
        const size_t bytes = (size_t)B * sizeof(ualm_result_t) + (size_t)(ocx_[B] + ocy_[B]) * sizeof(double) + (size_t)B * sizeof(int32_t);
        if (bytes > cap_) {
            release();
            cudaError_t e = cudaHostAlloc(&h_, bytes, cudaHostAllocMapped);
            if (e == cudaSuccess) e = cudaHostGetDevicePointer(&d_, h_, 0);
            if (e != cudaSuccess) { release(); return e; }
            cap_ = bytes;
        }
        host_ = carve(h_);
        dev_ = carve(d_);
        memset(host_.flag, 0, sizeof(int32_t) * (size_t)B);
        for (int b = 0; b < B; b++) {
            if (!skip[b]) continue;
            memset(&host_.res[b], 0, sizeof(ualm_result_t));
            host_.res[b].ret_code = UALM_ELIMIT;
            memset(host_.c_xy + ocx_[b], 0, sizeof(double) * (size_t)(ocx_[b + 1] - ocx_[b]));
            memset(host_.c_yaw + ocy_[b], 0, sizeof(double) * (size_t)(ocy_[b + 1] - ocy_[b]));
            host_.flag[b] = 1;
        }
        return cudaSuccess;
    }

    // device view of the current batch (for the kernels that publish)
    const Ptrs &device() const { return dev_; }

    // Problems whose flag is up and that this ticket has not returned yet: their indices into idx (in problem order), their records
    // and coefficients into results / c_xy / c_yaw at their problem-order positions (any of the three may be null).  Returns how
    // many.
    int collect(int32_t *idx, ualm_result_t *results, double *c_xy, double *c_yaw)
    {
        int n = 0;
        for (int b = 0; b < B_; b++) {
            if (returned_[b] || __atomic_load_n(host_.flag + b, __ATOMIC_ACQUIRE) == 0) continue;
            if (results) memcpy(&results[b], &host_.res[b], sizeof(ualm_result_t));
            if (c_xy) memcpy(c_xy + ocx_[b], host_.c_xy + ocx_[b], sizeof(double) * (size_t)(ocx_[b + 1] - ocx_[b]));
            if (c_yaw) memcpy(c_yaw + ocy_[b], host_.c_yaw + ocy_[b], sizeof(double) * (size_t)(ocy_[b + 1] - ocy_[b]));
            returned_[b] = 1;
            idx[n++] = b;
        }
        n_returned_ += n;
        return n;
    }
    int pending() const { return B_ - n_returned_; }

    void release()
    {
        if (h_) cudaFreeHost(h_);
        h_ = d_ = nullptr;
        cap_ = 0;
        host_ = dev_ = Ptrs{};
    }

private:
    Ptrs carve(void *base) const
    {
        Ptrs p;
        char *q = (char *)base;
        p.res = (ualm_result_t *)q;            q += (size_t)B_ * sizeof(ualm_result_t);
        p.c_xy = (double *)q;                  q += (size_t)ocx_[B_] * sizeof(double);
        p.c_yaw = (double *)q;                 q += (size_t)ocy_[B_] * sizeof(double);
        p.flag = (int32_t *)q;
        return p;
    }
    void *h_ = nullptr, *d_ = nullptr;
    size_t cap_ = 0;
    int B_ = 0, n_returned_ = 0;
    std::vector<long long> ocx_, ocy_;
    std::vector<unsigned char> returned_;
    Ptrs host_{}, dev_{};
};

} // namespace ualm_mbox
