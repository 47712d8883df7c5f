// api.h -- what every C ABI entry point shares: the error message pvb_last_error returns, and the workspace check.
// Each op's entry points live at the end of its own .cu file; the voting layer's are in api.cu.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "../../include/pvnet_vote_b200.h"

namespace pvb {

// records the message for pvb_last_error and returns `code`
int fail(int code, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
// PVB_ERR_CUDA with "<what>: <the CUDA error string>"
int cuda_fail(cudaError_t e, const char *what);

inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

// the caller's device workspace of `bytes` at `ws` against the `need` bytes of the call: NULL is fine when need == 0,
// otherwise it must hold `need` bytes and be 256-byte aligned (PVB_ERR_WORKSPACE)
int check_workspace(size_t need, const void *ws, size_t bytes);

} // namespace pvb
