// incr.cu -- ONE launch for the evaluation an MCMC chain issues almost every step (MarkovChain.java:207-393: a move
// dirties one or two root paths): updateTransitionMatrices (a few branches) -> updatePartials (a short list) ->
// calculateRootLogLikelihoods.  Through separate launches that sequence costs three to five dependent launches, three
// staged H2D copies and a D2H copy + stream synchronise -- ~60 us for ~13 ops of which the GPU computes ~15 us.
//
// The host defers the first two calls when the list is short (api.cu, "deferred small evaluations") and this kernel
// does all of it, everything travelling BY VALUE in the kernel parameters (no staging copies):
//   0. every block recomputes the pending branches' spectra exp(lambda_k r_c t) and P(t) into shared memory (a few
//      hundred flops -- cheaper than a grid-wide dependency on a matrix kernel); block 0 also writes them to HBM in all
//      the layouts later launches read (exactly what k_transition4 writes);
//   1. the op list in eigen form, one (pattern, category) cell per thread, the previous op's result forwarded in registers;
//   2. the root integration on the last op's result while it is still in registers: categories meet through warp shuffles,
//      site log-likelihoods are stored, the weighted sum is reduced across blocks (fixed order) and the finishing block
//      writes the value into MAPPED PINNED host memory followed by a sequence flag -- the host spins on the flag, no
//      cudaMemcpy, no cudaStreamSynchronize.
// Lists the form does not cover are flushed through the ordinary path (nothing is lost, only the fusion).
#include "engine.h"
#include "walk4.cuh"

namespace b200 {

namespace {

__device__ __forceinline__ double absBitsI(double v) {
    return __hiloint2double(__double2hiint(v) & 0x7fffffff, __double2loint(v));
}

template <typename T, int CP>
__device__ __forceinline__ void incrementalBody(const IncArgs& A) {
    constexpr int G = 32 / CP;
    __shared__ double sE[kIncMaxMats][CP][4];
    __shared__ __align__(16) double sP[kIncMaxMats][CP][16];      // [c][j][i]: column j of P_c = contribution of a tip in state j
    __shared__ double red[4];
    __shared__ bool last;
    const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
    const int S = A.S, C = A.C;
    const int c = lane / G;
    const int p = blockIdx.x * (4 * G) + wib * G + (lane % G);
    const bool catValid = c < C;
    const int cc = catValid ? c : 0;
    const bool inRange = p < A.Ppad;
    const int pp = inRange ? p : 0;
    const size_t off0 = ((size_t)cc * A.Ppad + pp) * 4;
    // everything the chain will read from memory is known up front (the list is in the kernel parameters): start all of it
    // on its way to L1 FIRST, so that the HBM/L2 latency of the siblings' partials overlaps the matrix prelude below and the
    // dependent chain runs at cache-hit latency instead of one memory round trip per op
    for (int k = 0; k < A.nOps; ++k) {
        const IncOp op = A.op[k];
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
            const int child = ch == 0 ? op.c1 : op.c2, m = ch == 0 ? op.m1 : op.m2;
            if (child < 0) {
                if (c == 0) prefetchL1(A.states + (size_t)(-child - 1) * A.Ppad + pp);
                if (m >= 0 && lane < 4) prefetchL1(A.mats + (size_t)m * A.matStride + lane * 4 * CP);
            } else {
                if (!(ch == 0 && (op.flags & 1)) && catValid)
                    prefetchL1(static_cast<const T*>(A.partials) + (size_t)child * A.stride + off0);
                if (m >= 0 && lane == 0) prefetchL1(A.evecs + (size_t)m * CP * 4);
            }
        }
        if (op.sr >= 0 && c == 0) prefetchL1(A.scale + (size_t)op.sr * A.Ppad + pp);
    }
    if (c == 0) {
        prefetchL1(A.patternWeights + pp);
        if (A.cum != nullptr) prefetchL1(A.cum + pp);
    }
    // ---- 0. pending branches: spectra, then P = | V diag(e) V^-1 | with the reference's summation order
    for (int idx = tid; idx < A.nMats * C * 4; idx += 128) {
        const int q = idx / (C * 4), c = (idx >> 2) % C, k = idx & 3;
        sE[q][c][k] = k < S ? exp(A.eval[k] * A.rate[q][c] * A.mat[q].len) : 0.0;
    }
    __syncthreads();
    for (int idx = tid; idx < A.nMats * C * 16; idx += 128) {
        const int q = idx / (C * 16), c = (idx >> 4) % C, j = (idx >> 2) & 3, i = idx & 3;
        double acc = 0.0;
        if (i < S && j < S) {
#pragma unroll
            for (int k = 0; k < 4; ++k) acc += A.V[4 * i + k] * (sE[q][c][k] * A.Vi[4 * k + j]);
            acc = fabs(acc);
        }
        sP[q][c][j * 4 + i] = acc;
        if (blockIdx.x == 0) {             // the HBM copies every later launch reads (same layouts as k_transition4)
            double* base = A.mats + (size_t)A.mat[q].prob * A.matStride;
            base[((size_t)j * CP + c) * 4 + i] = acc;
            if (j == 0) A.evecs[((size_t)A.mat[q].prob * CP + c) * 4 + i] = sE[q][c][i];
        }
    }
    __syncthreads();

    // ---- 1. the list
    double d[4] = {0.0, 0.0, 0.0, 0.0};
    for (int k = 0; k < A.nOps; ++k) {
        const IncOp op = A.op[k];
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
            const int child = ch == 0 ? op.c1 : op.c2, m = ch == 0 ? op.m1 : op.m2;
            double y[4];
            if (child < 0) {
                const int s = (int)__ldg(A.states + (size_t)(-child - 1) * A.Ppad + pp);
                if (s < S) {
                    if (m < 0) {
                        const double* col = &sP[-m - 1][cc][s * 4];
                        y[0] = col[0]; y[1] = col[1]; y[2] = col[2]; y[3] = col[3];
                    } else {
                        ldg256_ro(A.mats + (size_t)m * A.matStride + ((size_t)s * CP + cc) * 4, y);
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 4; ++i) y[i] = (i < S) ? 1.0 : 0.0;
                }
            } else {
                double e[4], x[4], u[4];
                if (m < 0) { e[0] = sE[-m - 1][cc][0]; e[1] = sE[-m - 1][cc][1]; e[2] = sE[-m - 1][cc][2]; e[3] = sE[-m - 1][cc][3]; }
                else ldg256_ro(A.evecs + ((size_t)m * CP + cc) * 4, e);
                if (ch == 0 && (op.flags & 1)) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) x[i] = d[i];
                } else {
                    loadCell(static_cast<const T*>(A.partials) + (size_t)child * A.stride + off0, x);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    u[q] = (A.Vi[4 * q] * x[0] + A.Vi[4 * q + 1] * x[1] + A.Vi[4 * q + 2] * x[2] + A.Vi[4 * q + 3] * x[3]) * e[q];
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    y[i] = absBitsI(A.V[4 * i] * u[0] + A.V[4 * i + 1] * u[1] + A.V[4 * i + 2] * u[2] + A.V[4 * i + 3] * u[3]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) d[i] = ch == 0 ? y[i] : d[i] * y[i];
        }
        if (op.sw >= 0) {                      // rescaling, as in the walk kernels
            double mx = catValid ? fmax(fmax(d[0], d[1]), fmax(d[2], d[3])) : 0.0;
#pragma unroll
            for (int sh = G; sh < 32; sh <<= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, sh));
            if (mx == 0.0) mx = 1.0;
            const double inv = 1.0 / mx;
#pragma unroll
            for (int i = 0; i < 4; ++i) d[i] *= inv;
            if (c == 0 && inRange) A.scale[(size_t)op.sw * A.Ppad + p] = A.logScalers ? log(mx) : mx;
        } else if (op.sr >= 0) {
            double f = A.scale[(size_t)op.sr * A.Ppad + pp];
            if (A.logScalers) f = exp(f);
            const double inv = 1.0 / f;
#pragma unroll
            for (int i = 0; i < 4; ++i) d[i] *= inv;
        }
        roundCell<T>(d);                       // also what the next op and the root integration below read
        if (catValid && inRange) storeCell(static_cast<T*>(A.partials) + (size_t)op.dest * A.stride + off0, d);
    }

    // ---- 2. root: site[p] = log(sum_c w_c sum_i pi_i root[c,p,i]) + cum[p]; out = sum_p weight[p] site[p]
    double t = 0.0;
    if (catValid) t = A.weights[cc] * (A.freqs[0] * d[0] + A.freqs[1] * d[1] + A.freqs[2] * d[2] + A.freqs[3] * d[3]);
#pragma unroll
    for (int sh = G; sh < 32; sh <<= 1) t += __shfl_xor_sync(0xffffffffu, t, sh);
    double contrib = 0.0;
    if (c == 0 && p < A.P) {
        double s = log(t);
        if (A.cum != nullptr) s += A.cum[p];
        A.site[p] = s;
        contrib = A.patternWeights[p] * s;
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, sh);
    if (lane == 0) red[wib] = contrib;
    __syncthreads();
    if (tid == 0) {
        A.blockSums[blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);
        __threadfence();
        const unsigned done = atomicAdd(A.counter, 1u);
        last = (done == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        __threadfence();
        double acc = 0.0;
        for (int q = tid; q < (int)gridDim.x; q += 128) acc += A.blockSums[q];
#pragma unroll
        for (int sh = 16; sh > 0; sh >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sh);
        __syncthreads();
        if (lane == 0) red[wib] = acc;
        __syncthreads();
        if (tid == 0) {
            const double total = (red[0] + red[1]) + (red[2] + red[3]);
            *A.out = total;
            *A.counter = 0u;
            *A.hostOut = total;                          // mapped pinned memory: the value, then the flag
            __threadfence_system();
            *A.hostFlag = A.seq;
        }
    }
}

template <int CP>
__global__ void __launch_bounds__(128)
k_incremental(const IncArgs A) {
    incrementalBody<double, CP>(A);
}

// fp32 partials storage (PRECISION_SINGLE)
template <int CP>
__global__ void __launch_bounds__(128)
k_incrementals(const IncArgs A) {
    incrementalBody<float, CP>(A);
}

}  // namespace

cudaError_t launchIncremental(Instance* in, const IncArgs& A) {
    const int G = 32 / in->matCP;
    const int blocks = (in->Ppad + 4 * G - 1) / (4 * G);
    if (in->single) {
        switch (in->matCP) {
            case 1: k_incrementals<1><<<blocks, 128, 0, in->stream>>>(A); break;
            case 2: k_incrementals<2><<<blocks, 128, 0, in->stream>>>(A); break;
            case 4: k_incrementals<4><<<blocks, 128, 0, in->stream>>>(A); break;
            case 8: k_incrementals<8><<<blocks, 128, 0, in->stream>>>(A); break;
            default: return cudaErrorInvalidValue;
        }
        return cudaGetLastError();
    }
    switch (in->matCP) {
        case 1: k_incremental<1><<<blocks, 128, 0, in->stream>>>(A); break;
        case 2: k_incremental<2><<<blocks, 128, 0, in->stream>>>(A); break;
        case 4: k_incremental<4><<<blocks, 128, 0, in->stream>>>(A); break;
        case 8: k_incremental<8><<<blocks, 128, 0, in->stream>>>(A); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace b200
