// rexsim_host.h -- host-side plumbing shared by rexsim_capi.cu and rexsim_agent.cu (internal, no device code): the error
// string behind rexsim_last_error, the tail every launching entry point ends with, and the device memory a handle owns.
#pragma once
#include "../../include/rexsim.h"
#include <cuda_runtime.h>
#include <cstdio>
#include <vector>

namespace rexsim {

inline thread_local char g_err[512] = "";
inline int fail(int code, const char* msg) { snprintf(g_err, sizeof(g_err), "%s", msg); return code; }
inline int cuda_fail(cudaError_t e, const char* where) {
    snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
    return REXSIM_ERR_CUDA;
}
#define CK(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return rexsim::cuda_fail(_e, #x); } while (0)

// status of an entry point that has just launched: the CUDA error mapped, or the handle's launch counter advanced
template <class Handle>
int enqueue(Handle* h, cudaError_t e, const char* where, int launches = 1) {
    if (e != cudaSuccess) return cuda_fail(e, where);
    h->launches += launches;
    return REXSIM_OK;
}

// Every device allocation of a handle, so that destroy cannot forget one.
struct DeviceBuffers {
    std::vector<void*> ptrs;
    // *out = count zeroed elements; REXSIM_OK or REXSIM_ERR_CUDA (message set).  Ptr is deduced whole, so that the
    // __restrict__ pointer fields of a kernel's argument struct can be allocated in place.
    template <class Ptr>
    int zeroed(Ptr* out, size_t count) {
        void* p = nullptr;
        CK(cudaMalloc(&p, count * sizeof(**out)));
        ptrs.push_back(p);
        *out = static_cast<Ptr>(p);
        CK(cudaMemset(p, 0, count * sizeof(**out)));
        return REXSIM_OK;
    }
    // free one buffer of the list (a buffer that is reallocated with another size)
    void drop(void* p) {
        for (size_t i = 0; i < ptrs.size(); i++)
            if (ptrs[i] == p) { cudaFree(p); ptrs.erase(ptrs.begin() + i); return; }
    }
    void release() {
        for (void* p : ptrs) cudaFree(p);
        ptrs.clear();
    }
};

}  // namespace rexsim
