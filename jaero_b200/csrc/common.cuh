// jaero_b200 — shared host/device helpers (product code; sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <string>

namespace jb {

void set_error(const std::string &msg);          // capi.cu
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define JB_CUDA(call)                                                              \
    do {                                                                           \
        cudaError_t e_ = (call);                                                   \
        if (e_ != cudaSuccess) return jb::cuda_fail(e_, #call, __FILE__, __LINE__); \
    } while (0)

static const int WTSIZE = 19999;                 // JAERO/DSP.h:21

} // namespace jb
