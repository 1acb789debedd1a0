// clp_jit.h -- run-time compilation of the scoring kernel for a caller's CUDA-source invariant (clp_score_custom).
#pragma once
#include <string>

namespace clp {

// the kernels of clp_score_tile.cuh a caller's invariant is compiled into
enum class JitKernel { kScoreTile = 0, kBatchScore = 1 };

// kScoreTile: score_tile_kernel<T, 2, D, MIRROR> with the caller's clp_invariant, T = double if f64 else float;
// kBatchScore: batch_score_custom_kernel<D> (f64 and mirror are not used).  D = d for 1 <= d <= 16, else 0 (runtime
// d).  Compiled once per (kind, source, D, T, MIRROR, device) and kept for the life of the process; the kernel is loaded
// for `device`, which must be current.  Returns 0 and *fn (a handle for cudaLaunchKernel), CLP_ERR_INVALID with the
// compiler's log in *err when the source does not compile, or CLP_ERR_CUDA when the module cannot be loaded.
int jit_score_kernel(JitKernel kind, const std::string& source, int d, bool f64, bool mirror, int device, const void** fn,
                     std::string* err);

// compiles the fp32 / MIRROR instance for dimension d without loading it (no device needed); 0 or CLP_ERR_INVALID, the
// compiler's log in *log either way
int jit_check(const std::string& source, int d, std::string* log);

// NVRTC compilations of this process and their total wall-clock time in milliseconds
void jit_stats(long long* compiles, double* compile_ms);

}  // namespace clp
