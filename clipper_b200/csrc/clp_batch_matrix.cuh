// clp_batch_matrix.cuh -- many small problems given as (M, C) matrices, solved in ONE launch (clp_batch_solve_matrices).
//
// The counterpart of batch_solve_kernel for affinities the caller computed (a custom invariant, another consistency
// measure, a matrix read back with getAffinityMatrix): problem p arrives as two strictly-upper CSC matrices, exactly as
// clp_set_sparse_upper takes them, and gets what an fp32 handle gives after clp_set_sparse_upper + clp_solve.  One CTA
// of a persistent grid owns one problem (problems drawn from a counter):
//     neutral fill of the per-CTA fp32 scratch matrix -> scatter of the M entries, block barrier, scatter of the C
//     entries (the per-entry bodies of scatter_csc_M_kernel / scatter_csc_C_kernel) -> kept entries per row and the
//     plain test -> steps 3-4 of batch_solve_kernel (batch_build_solve): full-row sliced-ELL copy and the SOLO
//     resident solver
// The host has validated the input (structure, M >= 0, C in {0, 1}, rows strictly ascending) before the upload, so the
// flags the entry bodies raise stay clear.
#pragma once

namespace clp {

struct BatchMatProblem {    // device array, one per problem; offsets into the concatenated input / output arrays
  long long cpM_off, cpC_off;  // in int64: the problem's m + 1 column pointers (local: they start at 0)
  long long eM_off, eC_off;    // in entries: the problem's row indices and values
  long long u_off;             // in doubles: u0 in, final iterate out
  int m, pad_;
};

struct BatchMatArgs {
  const BatchMatProblem* prob;
  int nprob;
  const long long* colptr; const int* rowidx; const double* val;  // concatenated CSC arrays of all M and C matrices
  const double* u0;
  double* u_out;
  SolverOut* out;            // [nprob]
  unsigned int* nnz_out;     // [nprob] kept entries (i != j, both triangles)
  int* next;                 // problem counter
  unsigned long long* prof;  // nullable: [nprob][4] ns spent in fill+scatter+count, build, solve, whole problem
  unsigned char* scratch; size_t scratch_stride;
  int max_m;
  SolverParams prm;
  SyncBlock* sb;
  long long spin_limit;
};

__global__ void __launch_bounds__(kBatchThreads, 3) batch_matrix_solve_kernel(BatchMatArgs ba) {
  extern __shared__ __align__(128) unsigned char clp_batch_smem[];
  unsigned char* smem = clp_batch_smem;
  __shared__ ResArgs sa;
  __shared__ int s_p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const BatchLayout L = batch_layout(ba.max_m, 0, /*points*/ false);
  unsigned char* sc = ba.scratch + (size_t)blockIdx.x * ba.scratch_stride;
  float* M = reinterpret_cast<float*>(sc + L.M);
  unsigned int* rowid = reinterpret_cast<unsigned int*>(sc + L.rowid);
  unsigned int* itemptr = reinterpret_cast<unsigned int*>(sc + L.itemptr);
  unsigned int* ctafirst = reinterpret_cast<unsigned int*>(sc + L.ctafirst);
  float* val = reinterpret_cast<float*>(sc + L.val);
  unsigned short* idx = reinterpret_cast<unsigned short*>(sc + L.idx);

  for (;;) {
    __syncthreads();
    if (tid == 0) s_p = atomicAdd(ba.next, 1);
    __syncthreads();
    const int p = s_p;
    if (p >= ba.nprob) break;
    const BatchMatProblem P = ba.prob[p];
    const unsigned long long t_begin = global_ns();
    const int m = P.m;
    const int ld = (m + 127) / 128 * 128;
    const int rows_pad = (m + 3) / 4 * 4;
    const int NI = rows_pad / 4;
    const BatchSmem bs = batch_smem_plan(ba.max_m);
    unsigned int* cnt = reinterpret_cast<unsigned int*>(smem + bs.cnt);  // [rows_pad]

    // ---- 1. neutral fill: every element "no affinity, no constraint" (-0.0), padding rows and columns included
    {
      const float4 neutral4 = make_float4(-0.0f, -0.0f, -0.0f, -0.0f);
      float4* M4 = reinterpret_cast<float4*>(M);
      const size_t n4 = (size_t)rows_pad * ld / 4;
      for (size_t q = tid; q < n4; q += kBatchThreads) M4[q] = neutral4;
    }
    __syncthreads();
    // ---- 2. scatter, one warp per column: the M entries, then the C entries (a C bit is set on the stored affinity)
    for (int pass = 0; pass < 2; ++pass) {
      const long long* cp = ba.colptr + (pass ? P.cpC_off : P.cpM_off);
      const long long e0 = pass ? P.eC_off : P.eM_off;
      const int* ri = ba.rowidx + e0;
      const double* vv = ba.val + e0;
      for (int j = warp; j < m; j += kBatchWarps) {
        const long long q1 = cp[j + 1];
        for (long long q = cp[j] + lane; q < q1; q += 32) {
          if (pass == 0) scatter_csc_M_entry<float>(ri[q], j, vv + q, M, ld, 0, m, &ba.sb->flags);
          else scatter_csc_C_entry<float>(ri[q], j, vv + q, M, ld, 0, m, &ba.sb->flags);
        }
      }
      __syncthreads();
    }
    // ---- 3. kept entries of every row into cnt, and the plain test: every kept entry has M > 0 and C = 1
    unsigned int odd = 0;
    for (int i = warp; i < rows_pad; i += kBatchWarps) {
      unsigned int kept = 0;
      for (int j0 = lane * 4; j0 < ld; j0 += 128) {
        const float4 x = *reinterpret_cast<const float4*>(M + (size_t)i * ld + j0);
        const float xe[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (!is_neutral<float>(xe[e])) { ++kept; odd |= is_plain<float>(xe[e]) ? 0u : 1u; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
      if (lane == 0) cnt[i] = kept;
    }
    const int plain = __syncthreads_or((int)odd) ? 0 : 1;

    const unsigned long long t_scattered = global_ns();
    // ---- 4. full-row sliced-ELL copy and the solver, as for scored problems
    batch_build_solve(p, m, ld, rows_pad, NI, P.u_off, plain, M, rowid, itemptr, ctafirst, val, idx, sc, L, smem, bs, cnt,
                      ba.nnz_out, ba.prm, ba.u0, ba.u_out, ba.out, ba.sb, ba.spin_limit, ba.prof, t_begin, t_scattered, sa);
  }
}

}  // namespace clp
