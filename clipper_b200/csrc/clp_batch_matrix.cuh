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

// ---- dense device tensors (clp_batch_solve_dense_dev) -------------------------------------------------------------
// Problem p is the leading m x m block of [nprob, m_max, m_max] tensors in HBM: entry (i, j) at
// base[p * bstride + i * rs + j * cs] (one of rs, cs is 1); only its strict upper triangle is read.  In place of steps 1-3
// of batch_matrix_solve_kernel, one pass over the tile pairs of the padded square (ld x ld) stores every element of the
// scratch's rows_pad x ld block exactly once (dense_entry above the diagonal and its mirror below it, neutral on the
// diagonal and in the padding) and counts the kept entries of every row and the plain test on the way.  A problem with
// a negative M or a C outside {0, 1} is neither built nor solved; the lowest such problem (M errors first) is left in
// *bad as ((3 - kind) << 32 | ~p), the largest key winning (kind 1: M, 2: C).
struct BatchDenseArgs {
  const BatchMatProblem* prob;   // m and u_off of every problem
  int nprob;
  const void* M; const void* C;  // In[nprob][..][..] as described above
  long long bstride, rs, cs;
  const double* u0_in; long long u0_stride;  // the caller's u0, row p at p * u0_stride
  double* u0;                                // staged u0 (u_off), what the solver reads
  double* u_out;                             // final iterates (u_off), read back by the host
  double* u_out_dev; long long u_out_stride;  // nullable: the caller's copy of them
  SolverOut* out;
  unsigned int* nnz_out;
  int* next;
  unsigned long long* bad;
  unsigned long long* prof;      // nullable: [nprob][4] ns spent in load+count, build, solve, whole problem
  unsigned char* scratch; size_t scratch_stride;
  int max_m;
  SolverParams prm;
  SyncBlock* sb;
  long long spin_limit;
};

template <typename In>
__global__ void __launch_bounds__(kBatchThreads, 3) batch_dense_solve_kernel(BatchDenseArgs ba) {
  extern __shared__ __align__(128) unsigned char clp_batch_smem[];
  unsigned char* smem = clp_batch_smem;
  __shared__ ResArgs sa;
  __shared__ int s_p;
  const int tid = threadIdx.x, lane = tid & 31;
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
    // the tile overlays the scoring queue and tile regions (6 KB), unused by a given-matrix problem
    float (*sh)[33] = reinterpret_cast<float (*)[33]>(smem + bs.queue);
    const In* Mg = reinterpret_cast<const In*>(ba.M) + (size_t)p * ba.bstride;
    const In* Cg = reinterpret_cast<const In*>(ba.C) + (size_t)p * ba.bstride;

    for (int i = tid; i < rows_pad; i += kBatchThreads) cnt[i] = 0u;
    for (int i = tid; i < m; i += kBatchThreads) ba.u0[P.u_off + i] = ba.u0_in[(size_t)p * ba.u0_stride + i];
    __syncthreads();
    // ---- 1. load: tile pairs (bi <= bj) of the ld x ld square; each element of rows < rows_pad stored once
    unsigned int bad = 0, odd = 0;
    const int nt = ld / 32;
    for (int bj = 0; bj < nt; ++bj) {
      for (int bi = 0; bi <= bj; ++bi) {
        const int i0 = bi * 32, j0 = bj * 32;
        dense_tile_load<float, In>(Mg, Cg, ba.rs, ba.cs, m, i0, j0, sh, bad);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int k = (tid >> 5) + 8 * q;
          // row i0 + k: the tile's row (on a diagonal tile: upper part from the row, lower part from the column)
          const float a = (bi != bj || lane > k) ? sh[k][lane] : sh[lane][k];
          const bool ka = !is_neutral<float>(a);
          odd |= (ka && !is_plain<float>(a)) ? 1u : 0u;
          const unsigned int na = __popc(__ballot_sync(0xffffffffu, ka));
          if (i0 + k < rows_pad) {
            M[(size_t)(i0 + k) * ld + j0 + lane] = a;
            if (lane == 0 && na) atomicAdd(&cnt[i0 + k], na);
          }
          if (bi != bj) {  // row j0 + k: the tile's column k (the mirror)
            const float b = sh[lane][k];
            const bool kb = !is_neutral<float>(b);
            odd |= (kb && !is_plain<float>(b)) ? 1u : 0u;
            const unsigned int nb = __popc(__ballot_sync(0xffffffffu, kb));
            if (j0 + k < rows_pad) {
              M[(size_t)(j0 + k) * ld + i0 + lane] = b;
              if (lane == 0 && nb) atomicAdd(&cnt[j0 + k], nb);
            }
          }
        }
        __syncthreads();
      }
    }
    const int bad_m = __syncthreads_or((int)(bad & 1u));
    const int bad_c = __syncthreads_or((int)(bad & 2u));
    const int plain = __syncthreads_or((int)odd) ? 0 : 1;
    if (bad_m || bad_c) {
      if (tid == 0) atomicMax(ba.bad, ((unsigned long long)(bad_m ? 2u : 1u) << 32) | (0xffffffffu - (unsigned int)p));
      continue;
    }

    const unsigned long long t_loaded = global_ns();
    // ---- 2. full-row sliced-ELL copy and the solver, as for scored problems
    batch_build_solve(p, m, ld, rows_pad, NI, P.u_off, plain, M, rowid, itemptr, ctafirst, val, idx, sc, L, smem, bs, cnt,
                      ba.nnz_out, ba.prm, ba.u0, ba.u_out, ba.out, ba.sb, ba.spin_limit, ba.prof, t_begin, t_loaded, sa);
    if (ba.u_out_dev) {  // the problem is read again rather than kept in registers across the solver
      __syncthreads();
      const int q = s_p;
      const BatchMatProblem Q = ba.prob[q];
      for (int i = tid; i < Q.m; i += kBatchThreads) ba.u_out_dev[(size_t)q * ba.u_out_stride + i] = __ldcg(ba.u_out + Q.u_off + i);
    }
  }
}

}  // namespace clp
