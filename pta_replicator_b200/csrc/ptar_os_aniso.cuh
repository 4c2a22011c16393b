// Anisotropy of the optimal statistic (ptar_os_aniso): spherical-harmonic fits and radiometer sky maps of every
// realization, from the per-pulsar projections X that os_sum wrote.
//
// Every output is a fixed, realization-independent linear map of the pair correlations d_q = x_a . x_b
// (engine.PulsarBatch._plan_os_aniso), so the whole map is one GEMM with ptar_os_null's sky-scramble operands:
//   map[r][c] = (sum_q U[r][q] V[q][c]) / dsqrt[c],   U[r][q] = x_a . x_b,   x = X phi~^{1/2},  q = (a < b) of os.pairs
//   columns c = [ c^_lm (n_lm) | z (n_z = n_lm - 1) | radiometer S/N_k (n_sky) ]
// Stages 1-2 launch os_null_prepare_kernel and os_null_gemm_kernel on a ptar_os_null_model view of the model.
// os_aniso_reduce  one CTA per realization: copies c^ and z, chi2 = sum z^2 by a fixed tree, (max, first argmax) of the
//                  radiometer S/N by a fixed tree (ties to the lower pixel, the first NaN above every number, as
//                  fe_better), and the S/N map only when the caller asks for it.  No atomics: every output is
//                  bit-identical whatever nreal, chunking or real0.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ptar.h"
#include "ptar_fe.cuh"
#include "ptar_os_null.cuh"

namespace ptar {

constexpr int AN_THREADS = 256;
static_assert(PTAR_OS_ANISO_MAX_LM <= AN_THREADS, "one z component per thread: the chi2 tree order is fixed by z's index");

__global__ void __launch_bounds__(AN_THREADS) os_aniso_reduce_kernel(const double* __restrict__ map, ptar_os_aniso_model am,
                                                                     double* __restrict__ clm, double* __restrict__ z,
                                                                     double* __restrict__ chi2, double* __restrict__ snr_max,
                                                                     int64_t* __restrict__ argmax,
                                                                     double* __restrict__ radio_map) {
  __shared__ double sv[AN_THREADS];
  __shared__ int si[AN_THREADS];
  const int64_t r = blockIdx.x;
  const int tid = threadIdx.x;
  const double* row = map + r * am.n_col;
  if (am.n_lm > 0) {
    if (tid < am.n_lm) clm[r * am.n_lm + tid] = row[tid];
    double s = 0.0;
    if (tid < am.n_z) {
      const double v = row[am.n_lm + tid];
      z[r * am.n_z + tid] = v;
      s = __dmul_rn(v, v);
    }
    sv[tid] = s;
    __syncthreads();
    for (int h = AN_THREADS / 2; h > 0; h >>= 1) {
      if (tid < h) sv[tid] = __dadd_rn(sv[tid], sv[tid + h]);
      __syncthreads();
    }
    if (tid == 0) chi2[r] = sv[0];
    __syncthreads();
  }
  if (am.n_sky > 0) {
    const double* sr = row + am.n_lm + am.n_z;
    double* mr = radio_map ? radio_map + r * am.n_sky : nullptr;
    double best = -INFINITY;
    int bi = INT32_MAX;   // ranks below every pixel: a -inf pixel still wins on its index
    for (int k = tid; k < am.n_sky; k += AN_THREADS) {
      const double v = sr[k];
      if (mr) mr[k] = v;
      if (fe_better(v, k, best, bi)) {
        best = v;
        bi = k;
      }
    }
    sv[tid] = best;
    si[tid] = bi;
    __syncthreads();
    for (int h = AN_THREADS / 2; h > 0; h >>= 1) {
      if (tid < h && fe_better(sv[tid + h], si[tid + h], sv[tid], si[tid])) {
        sv[tid] = sv[tid + h];
        si[tid] = si[tid + h];
      }
      __syncthreads();
    }
    if (tid == 0) {
      snr_max[r] = sv[0];
      argmax[r] = si[0];
    }
  }
}

}  // namespace ptar
