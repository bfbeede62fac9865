// kernels.cu -- hand-written sm_90a kernels of the tree-likelihood hot path.
//
//   k_transition4  : P_c(t) = Evec diag(exp(Eval r_c t)) Ievc, 4-state layouts (updateTransitionMatrices)
//   k_transition   : the same for the generic layout when k_transition_mma does not apply
//   k_walk4        : 4-state (nucleotide) partials, WARP-OWNED PATTERN COLUMNS walking the whole
//                    operation list on-device; per-thread shared-memory operand stack (updatePartials)
//   k_walk_generic : any state count, BLOCK-OWNED pattern tiles walking the list  (updatePartials)
//   k_root         : frequency/category integration + log + scalers + weighted reduction
//   k_scale_accum  : cumulative scale buffers
//
// Why "walk": Felsenstein pruning has no cross-pattern data flow.  A pattern column (all categories
// and states of one site pattern) of a parent depends only on the same column of its children, so a
// warp (or block) that owns a set of columns can execute the ENTIRE post-order operation list for
// them without any grid-wide synchronisation: one launch per updatePartials call instead of one per
// node, and children produced earlier in the same list are read back from shared memory (the
// operand stack), not from HBM.  The only mandatory HBM traffic is the write of every destination
// buffer (BEAST needs them for later incremental updates) plus tips and pre-existing siblings.
#include "engine.h"
#include "walk4.cuh"

#include <algorithm>
#include <cfloat>

namespace b200 {

// fp64 tensor-core primitive (SASS DMMA.8x8x4): D(8x8) += A(8x4) * B(4x8); lane (g = lane/4, t = lane%4)
// holds A[g][t], B[t][g] and D[g][2t], D[g][2t+1]
__device__ __forceinline__ void dmma884acc(double& d0, double& d1, double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
        : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// ---------------------------------------------------------------------------------------------
// transition matrices
// ---------------------------------------------------------------------------------------------
// generic layout (matCP == 0).  grid (count, C); dynamic smem: ec[S], ss[S], pt[S](int).  Follows
// BaseSubstitutionModel.java:206-241 (real) / ComplexColtEigenSystem.java:71-139 (2x2 blocks), abs() convention; output
// TRANSPOSED.
__global__ void k_transition(const double* __restrict__ eigenBase, size_t eigenStride, int S, int Sp, int C,
                             int complexForm, const double* __restrict__ ratesBase,
                             const int* __restrict__ probIdx, const int* __restrict__ eigenIdx,
                             const int* __restrict__ rateSet, const double* __restrict__ lengths,
                             double* __restrict__ matBase, size_t matStride) {
    extern __shared__ double sm[];
    double* ec = sm;
    double* ss = sm + S;
    int* pt = reinterpret_cast<int*>(sm + 2 * S);
    const int b = blockIdx.x, c = blockIdx.y;
    const double* E = eigenBase + (size_t)eigenIdx[b] * eigenStride;
    const double* evec = E;
    const double* ievc = E + (size_t)S * S;
    const double* eval = E + 2 * (size_t)S * S;
    const double d = lengths[b] * ratesBase[(size_t)rateSet[b] * C + c];
    for (int k = threadIdx.x; k < S; k += blockDim.x) {
        double im = complexForm ? eval[S + k] : 0.0;
        if (im == 0.0) {
            ec[k] = exp(d * eval[k]); ss[k] = 0.0; pt[k] = k;
        } else {
            // rows of a conjugate pair are adjacent; the FIRST row's imaginary part drives the block
            // robust pairing: count consecutive non-zero imaginary rows above k
            int run = 0;
            for (int q = k - 1; q >= 0 && eval[S + q] != 0.0; --q) ++run;
            const bool first = (run % 2 == 0);
            int k0 = first ? k : k - 1;
            double bb = eval[S + k0];
            double expat = exp(d * eval[k0]);
            ec[k] = expat * cos(d * bb);
            ss[k] = (first ? 1.0 : -1.0) * expat * sin(d * bb);
            pt[k] = first ? k + 1 : k - 1;
        }
    }
    __syncthreads();
    // [c][j][i]
    double* out = matBase + (size_t)probIdx[b] * matStride + (size_t)c * Sp * Sp;
    for (int idx = threadIdx.x; idx < Sp * Sp; idx += blockDim.x) {
        int j = idx / Sp, i = idx % Sp;          // out[j][i] = P[i][j]
        double acc = 0.0;
        if (i < S && j < S) {
            for (int k = 0; k < S; ++k) {
                double iexp = ec[k] * ievc[(size_t)k * S + j] + ss[k] * ievc[(size_t)pt[k] * S + j];
                acc += evec[(size_t)i * S + k] * iexp;
            }
            acc = fabs(acc);
        }
        out[(size_t)j * Sp + i] = acc;
        // second half of the buffer holds the row-major M[c][i][j] (tensor-path B operand)
        const size_t ld = (size_t)Sp + 4;
        double* padded = matBase + (size_t)probIdx[b] * matStride + (size_t)C * Sp * Sp;
        padded[((size_t)c * Sp + i) * ld + j] = acc;                                   // M[c][i][.]
        padded[(size_t)C * Sp * ld + ((size_t)c * Sp + j) * ld + i] = acc;             // MT[c][j][.]
    }
}

// 4-state layout (matCP > 0, Sp == 4).  One quad of lanes per (branch, category), kTransition4Block-thread blocks over
// count x C quads.  The branch records (length and the matrix, eigen and rate-set indices) are read where the host staged
// them, in pinned memory over PCIe: the first threads of a block fetch the block's few contiguous records into shared
// memory once, so that every record crosses the bus in a handful of wide requests instead of once per warp that uses it.
// Lane k of a quad forms exp(d lambda_k) -- and for a complex pair the cos/sin terms and the partner row pt -- with
// k_transition's expressions and hands them to the other three lanes by shuffle.  Lane k = 2g + h then forms the 2 x 2 tile
// P[2h..2h+1][2g..2g+1]: that way each 16-byte store of the quad fills whole 32-byte sectors in every copy below (row-major
// P and its transpose alike), where a lane holding a whole row would write each sector in two halves.  Every product and
// sum is an explicit _rn operation in the order k_transition compiles to (iexp = fma(ec_m, Ievc[m][j], ss_m * Ievc[pt_m][j]),
// acc = fma(Evec[i][m], iexp, acc) from +0, m ascending), so both give the same bits and ptxas cannot contract otherwise.
// Writes, per (branch, category):
//   [j][CP][i]    : row j of all categories is one 128-byte line (k_walk4*, k_walk4e matrix form, getTransitionMatrix)
//   [matrix][CP][4] spectrum exp(lambda_k r_c t) for the eigen-form walk (walk4e.cu)
//   Mpad[c][8][4] : B fragment of k_walk4t, lane (g,t) reads [g][t]; rows g >= 4 stay zero
//   MTg [c][5][4] : column s of P for a compact tip in state s, plus the gap column s == S = (1,..,1,0..)
constexpr int kTransition4Block = 256;
__global__ void __launch_bounds__(kTransition4Block)
k_transition4(const double* __restrict__ eigenBase, size_t eigenStride, int S, int C, int CP, int complexForm,
              const double* __restrict__ ratesBase, const int* __restrict__ probIdx, const int* __restrict__ eigenIdx,
              const int* __restrict__ rateSet, const double* __restrict__ lengths, int count,
              double* __restrict__ matBase, size_t matStride, double* __restrict__ evecBase) {
    constexpr int Q = kTransition4Block / 4;                      // quads per block: at most Q branches (C = 1)
    __shared__ double sLen[Q];
    __shared__ int sProb[Q], sEig[Q], sRate[Q];
    const int lane = threadIdx.x & 31, k = lane & 3, i0 = 2 * (k & 1), j0 = 2 * (k >> 1);   // tile rows i0.., columns j0..
    const unsigned quad = 0xFu << (lane & ~3);
    const int q = (int)(blockIdx.x * (unsigned)Q + (threadIdx.x >> 2));
    const int bFirst = (int)(blockIdx.x * (unsigned)Q) / C;
    const int nb = min(count, ((int)(blockIdx.x * (unsigned)Q) + Q - 1) / C + 1) - bFirst;
    if ((int)threadIdx.x < nb) {
        sLen[threadIdx.x] = lengths[bFirst + threadIdx.x];
        sProb[threadIdx.x] = probIdx[bFirst + threadIdx.x];
        sEig[threadIdx.x] = eigenIdx[bFirst + threadIdx.x];
        sRate[threadIdx.x] = rateSet[bFirst + threadIdx.x];
    }
    __syncthreads();
    if (q >= count * C) return;                                   // whole quads leave together
    const int b = q / C, c = q - b * C, r = b - bFirst;
    const double* E = eigenBase + (size_t)sEig[r] * eigenStride;
    const double* evec = E;
    const double* ievc = E + (size_t)S * S;
    const double* eval = E + 2 * (size_t)S * S;
    const double d = __dmul_rn(sLen[r], ratesBase[(size_t)sRate[r] * C + c]);
    // the tile's rows of Evec and columns of Ievc do not depend on the exponentials: in flight while those are formed
    double V[2][4], W[4][2];
#pragma unroll
    for (int m = 0; m < 4; ++m)
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            V[t][m] = (i0 + t < S && m < S) ? evec[(size_t)(i0 + t) * S + m] : 0.0;
            W[m][t] = (m < S && j0 + t < S) ? ievc[(size_t)m * S + j0 + t] : 0.0;
        }
    double ec = 0.0, ss = 0.0;
    int pt = k;
    if (k < S) {
        const double im = complexForm ? eval[S + k] : 0.0;
        if (im == 0.0) {
            ec = exp(__dmul_rn(d, eval[k]));
        } else {
            // rows of a conjugate pair are adjacent; the FIRST row's imaginary part drives the block
            int run = 0;
            for (int m = k - 1; m >= 0 && eval[S + m] != 0.0; --m) ++run;
            const bool first = (run % 2 == 0);
            const int k0 = first ? k : k - 1;
            const double bb = eval[S + k0];
            const double expat = exp(__dmul_rn(d, eval[k0]));
            ec = __dmul_rn(expat, cos(__dmul_rn(d, bb)));
            ss = __dmul_rn(__dmul_rn(first ? 1.0 : -1.0, expat), sin(__dmul_rn(d, bb)));
            pt = first ? k + 1 : k - 1;
        }
    }
    double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};                  // acc[a][t] = P[i0 + a][j0 + t] before abs()
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        const double ecm = __shfl_sync(quad, ec, m, 4);
        const double ssm = __shfl_sync(quad, ss, m, 4);
        const int ptm = __shfl_sync(quad, pt, m, 4);
        if (m < S) {
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                // the partner row of a complex pair is read where k_transition reads it
                const double wp = (ptm == m || j0 + t >= S) ? W[m][t] : ievc[(size_t)ptm * S + j0 + t];
                const double iexp = __fma_rn(ecm, W[m][t], __dmul_rn(ssm, wp));
#pragma unroll
                for (int a = 0; a < 2; ++a) acc[a][t] = __fma_rn(V[a][m], iexp, acc[a][t]);
            }
        }
    }
    double p[2][2], g[2][2];                                      // the tile after abs(); the same as MTg entries [j][i]
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int i = i0 + a, j = j0 + t;
            p[a][t] = (i < S && j < S) ? fabs(acc[a][t]) : 0.0;
            g[a][t] = (j < S) ? p[a][t] : ((j == S && i < S) ? 1.0 : 0.0);
        }
    const int mat = sProb[r];
    double* base = matBase + (size_t)mat * matStride;
    double* mm = base + 16 * (size_t)CP + (size_t)c * 32;
    double* mt = base + 16 * (size_t)CP + (size_t)C * 32 + (size_t)c * 20;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
        // row j0 + t of [j][CP][i] and of MTg, entries i0, i0 + 1; row i0 + t of Mpad, entries j0, j0 + 1
        *reinterpret_cast<double2*>(base + ((size_t)(j0 + t) * CP + c) * 4 + i0) = make_double2(p[0][t], p[1][t]);
        *reinterpret_cast<double2*>(mt + (j0 + t) * 4 + i0) = make_double2(g[0][t], g[1][t]);
        *reinterpret_cast<double2*>(mm + (i0 + t) * 4 + j0) = make_double2(p[t][0], p[t][1]);
        *reinterpret_cast<double2*>(mm + 16 + 8 * t + 2 * k) = make_double2(0.0, 0.0);
    }
    mt[16 + k] = S == 4 ? 1.0 : 0.0;
    evecBase[((size_t)mat * CP + c) * 4 + k] = k < S ? ec : 0.0;
}

// convolveTransitionMatrices / addTransitionMatrices (SubstitutionModelDelegate.java:303-470, epoch and branch-specific
// models): result = first x second per category, resp. first + second, on the device, written in every layout the walk
// kernels read.  grid (pairs, C); the operands must not alias the result (the host falls back otherwise).
__device__ __forceinline__ size_t matEntry(int matCP, int Sp, int c, int i, int j) {      // P[c][i][j] in the canonical copy
    return matCP ? ((size_t)j * matCP + c) * 4 + i : ((size_t)c * Sp + j) * Sp + i;
}
__global__ void __launch_bounds__(256)
k_combine_matrices(double* __restrict__ matBase, size_t matStride, int S, int Sp, int C, int matCP,
                   const int* __restrict__ first, const int* __restrict__ second, const int* __restrict__ result, int multiply) {
    const int q = blockIdx.x, c = blockIdx.y;
    const double* A = matBase + (size_t)first[q] * matStride;
    const double* B = matBase + (size_t)second[q] * matStride;
    double* R = matBase + (size_t)result[q] * matStride;
    for (int idx = threadIdx.x; idx < Sp * Sp; idx += blockDim.x) {
        const int i = idx / Sp, j = idx % Sp;
        double v = 0.0;
        if (i < S && j < S) {
            if (multiply) for (int k = 0; k < S; ++k) v += A[matEntry(matCP, Sp, c, i, k)] * B[matEntry(matCP, Sp, c, k, j)];
            else v = A[matEntry(matCP, Sp, c, i, j)] + B[matEntry(matCP, Sp, c, i, j)];
        }
        R[matEntry(matCP, Sp, c, i, j)] = v;
        if (!matCP) {
            const size_t ld = (size_t)Sp + 4;
            double* padded = R + (size_t)C * Sp * Sp;
            padded[((size_t)c * Sp + i) * ld + j] = v;                                  // M[c][i][.]
            padded[(size_t)C * Sp * ld + ((size_t)c * Sp + j) * ld + i] = v;            // MT[c][j][.]
        } else {
            double* mm = R + 16 * matCP;                                                // tensor-variant copies (k_walk4t)
            mm[(size_t)c * 32 + i * 4 + j] = v;
            mm[(size_t)c * 32 + 16 + i * 4 + j] = 0.0;
            double* mt = mm + (size_t)C * 32;
            mt[(size_t)c * 20 + j * 4 + i] = (j < S) ? v : ((j == S && i < S) ? 1.0 : 0.0);
            if (j == 0) mt[(size_t)c * 20 + 16 + i] = (S == 4 && i < S) ? 1.0 : 0.0;
        }
    }
}

cudaError_t launchCombineMatrices(Instance* in, const int* dFirst, const int* dSecond, const int* dResult, int count, bool multiply) {
    if (count <= 0) return cudaSuccess;
    k_combine_matrices<<<dim3(count, in->C), 256, 0, in->stream>>>(in->dMat, in->matStride, in->S, in->Sp, in->C, in->matCP,
                                                                   dFirst, dSecond, dResult, multiply ? 1 : 0);
    return cudaGetLastError();
}

// Tensor-core variant for real eigen systems with S > 4: one block per (branch, category) computes
// P = Evec * (diag(exp(lambda r t)) * Ievc) as an Sp x Sp x Sp DMMA product.  Shared memory holds
// A = Evec [i][k] and Bt[j][k] = exp(.)_k * Ievc[k][j], both with the conflict-free (Sp+4) row stride.
template <int NT>
__global__ void __launch_bounds__(128)
k_transition_mma(const double* __restrict__ eigenBase, size_t eigenStride, int S, int C,
                 const double* __restrict__ ratesBase, const int* __restrict__ probIdx,
                 const int* __restrict__ eigenIdx, const int* __restrict__ rateSet,
                 const double* __restrict__ lengths, double* __restrict__ matBase, size_t matStride) {
    constexpr int Sp = 8 * NT;
    constexpr int LD = Sp + 4;
    extern __shared__ double smt[];
    double* As = smt;                 // Evec[i][k]
    double* Bt = smt + Sp * LD;       // Bt[j][k]
    double* ex = Bt + Sp * LD;        // exp(d * lambda_k)
    const int b = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
    const double* E = eigenBase + (size_t)eigenIdx[b] * eigenStride;
    const double* evec = E;
    const double* ievc = E + (size_t)S * S;
    const double* eval = E + 2 * (size_t)S * S;
    const double d = lengths[b] * ratesBase[(size_t)rateSet[b] * C + c];
    for (int k = tid; k < Sp; k += 128) ex[k] = k < S ? exp(d * eval[k]) : 0.0;
    __syncthreads();
    for (int q = tid; q < Sp * Sp; q += 128) {
        const int r = q / Sp, col = q % Sp;
        As[r * LD + col] = (r < S && col < S) ? evec[(size_t)r * S + col] : 0.0;                       // [i][k]
        // q walks Ievc row-major ([k][j]) so the global read is coalesced; the shared write is the transpose
        Bt[col * LD + r] = (r < S && col < S) ? ievc[(size_t)r * S + col] * ex[r] : 0.0;               // Bt[j][k]
    }
    __syncthreads();
    const int lane = tid & 31, w = tid >> 5, g = lane >> 2, t = lane & 3;
    double* outT = matBase + (size_t)probIdx[b] * matStride + (size_t)c * Sp * Sp;                     // MT[j][i]
    double* outR = matBase + (size_t)probIdx[b] * matStride + (size_t)C * Sp * Sp + (size_t)c * Sp * LD;  // M[i][.], stride LD
    double* outTp = outR + (size_t)C * Sp * LD;                                                            // MT[j][.], stride LD
    for (int mt = w; mt < NT; mt += 4) {             // 8-row tiles of the output
        double acc[NT][2];
#pragma unroll
        for (int n = 0; n < NT; ++n) { acc[n][0] = 0.0; acc[n][1] = 0.0; }
        const double* arow = As + (8 * mt + g) * LD + t;
        const double* brow = Bt + g * LD + t;
#pragma unroll 4
        for (int kc = 0; kc < Sp / 4; ++kc) {
            const double a = arow[4 * kc];
#pragma unroll
            for (int n = 0; n < NT; ++n) dmma884acc(acc[n][0], acc[n][1], a, brow[n * 8 * LD + 4 * kc]);
        }
        const int i = 8 * mt + g;
#pragma unroll
        for (int n = 0; n < NT; ++n) {
            const int j = 8 * n + 2 * t;
            const double v0 = fabs(acc[n][0]), v1 = fabs(acc[n][1]);
            *reinterpret_cast<double2*>(outR + (size_t)i * LD + j) = make_double2(v0, v1);
            outT[(size_t)j * Sp + i] = v0;
            outT[(size_t)(j + 1) * Sp + i] = v1;
            outTp[(size_t)j * LD + i] = v0;
            outTp[(size_t)(j + 1) * LD + i] = v1;
        }
    }
}

template <int NT>
static cudaError_t launchTransitionMmaT(Instance* in, const int* dProbIdx, const int* dEigenIdx, const int* dRateSet,
                                        const double* dLengths, int count) {
    constexpr int Sp = 8 * NT;
    const size_t smem = (2 * (size_t)Sp * (Sp + 4) + Sp) * sizeof(double);
    static_assert(Sp <= 64, "shared-memory budget");
    cudaError_t e = cudaFuncSetAttribute(k_transition_mma<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    dim3 grid(count, in->C);
    k_transition_mma<NT><<<grid, 128, smem, in->stream>>>(in->dEigen, 2 * (size_t)in->S * in->S + 2 * in->S, in->S, in->C,
                                                          in->dRates, dProbIdx, dEigenIdx, dRateSet, dLengths, in->dMat,
                                                          in->matStride);
    return cudaGetLastError();
}

cudaError_t launchTransitionMatrices(Instance* in, const int* dProbIdx, const int* dEigenIdx,
                                     const int* dRateSet, const double* dLengths, int count) {
    if (count <= 0) return cudaSuccess;
    if (in->matCP > 0) {
        const unsigned blocks = (unsigned)(((size_t)count * in->C * 4 + kTransition4Block - 1) / kTransition4Block);
        k_transition4<<<blocks, kTransition4Block, 0, in->stream>>>(in->dEigen, 2 * (size_t)in->S * in->S + 2 * in->S, in->S, in->C,
                                                      in->matCP, in->complexEigen ? 1 : 0, in->dRates, dProbIdx, dEigenIdx,
                                                      dRateSet, dLengths, count, in->dMat, in->matStride, in->dEvec);
        return cudaGetLastError();
    }
    if (in->genericMma && !in->complexEigen) {
        switch (in->Sp / 8) {
            case 1: return launchTransitionMmaT<1>(in, dProbIdx, dEigenIdx, dRateSet, dLengths, count);
            case 2: return launchTransitionMmaT<2>(in, dProbIdx, dEigenIdx, dRateSet, dLengths, count);
            case 3: return launchTransitionMmaT<3>(in, dProbIdx, dEigenIdx, dRateSet, dLengths, count);
            case 4: return launchTransitionMmaT<4>(in, dProbIdx, dEigenIdx, dRateSet, dLengths, count);
            case 8: return launchTransitionMmaT<8>(in, dProbIdx, dEigenIdx, dRateSet, dLengths, count);
            default: break;
        }
    }
    size_t smem = (size_t)in->S * (2 * sizeof(double) + sizeof(int)) + 16;
    int threads = in->Sp * in->Sp >= 1024 ? 256 : (in->Sp * in->Sp >= 128 ? 128 : 32);
    dim3 grid(count, in->C);
    k_transition<<<grid, threads, smem, in->stream>>>(in->dEigen, 2 * (size_t)in->S * in->S + 2 * in->S, in->S,
                                                      in->Sp, in->C, in->complexEigen ? 1 : 0, in->dRates,
                                                      dProbIdx, dEigenIdx, dRateSet, dLengths, in->dMat,
                                                      in->matStride);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// 4-state walk
// ---------------------------------------------------------------------------------------------
// Warp layout: CP categories (power of two >= C) x G = 32/CP consecutive patterns.  lane = c*G + g.
// Each thread owns the 4 states of one (pattern, category) cell = 32 contiguous bytes in [C][Ppad][4].
// Per op and warp the L1/LSU wavefront budget is what bounds this kernel once HBM writes are the only
// DRAM traffic, so every access is shaped to touch the fewest 128-byte lines:
//   * op record: 64 B, warp-uniform, four 128-bit loads; record k+2 is prefetched to L1, record k+1 read after the
//     arithmetic (R > 1) or one op ahead (R = 1); it also names what the NEXT op will read (look-ahead prefetch)
//   * matrices : layout [j][CP][i] -> row j of all categories is one 128-byte line, 4 loads per child
//   * the child produced by the previous op of the walk: taken from the thread's own registers (op flag bit 1);
//     optional variant (B200_WALK_VARIANT=1): a per-thread operand stack in shared memory for every such child,
//     laid out [slot][half][thread] so every LDS.128/STS.128 is bank-conflict free
//   * tip states: one byte per pattern; their line is prefetched one op ahead
struct Mat4 { double r[4][4]; };     // r[j][i] = P[i][j] of this thread's category

template <int CP>
__device__ __forceinline__ void loadMat(const double* __restrict__ m, Mat4& M) {
    ldg256_ro(m, M.r[0]); ldg256_ro(m + 4 * CP, M.r[1]); ldg256_ro(m + 8 * CP, M.r[2]); ldg256_ro(m + 12 * CP, M.r[3]);
}

__device__ __forceinline__ void applyMat(const Mat4& M, const double (&x)[4], double (&y)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) y[i] = M.r[0][i] * x[0] + M.r[1][i] * x[1] + M.r[2][i] * x[2] + M.r[3][i] * x[3];
}

// grid = (pattern tiles, subtrees of this phase).  Latency is hidden by thread-level parallelism
// (many independent (subtree, tile) walks per SM).  What bounds the kernel once DRAM only sees the
// mandatory writes is the LSU->register-file path (128 B/clk/SM): a 4x4 matrix costs every thread
// 128 B per child, more than the partials themselves, so each thread keeps its category's two
// matrices in registers and re-uses them for R patterns (R = patterns per thread, strided by G so
// that every load/store instruction still covers 8 consecutive patterns = 256 contiguous bytes).
// one child's contribution for the R patterns of this thread: y[r][i] (*)= sum_j P[i][j] x_r[j]
template <typename T, int CP, int R, bool STACK, bool FIRST>
__device__ __forceinline__ void childTerm(const WalkArgs& A, int child, int matIdx, int slot, int moff, size_t off0,
                                          int p0, bool catValid, int pBegin, int pEnd, const double2* stackMem,
                                          int nthreads, double (&y)[R][4]) {
    constexpr int G = 32 / CP;
    const int S = A.S;
    const double* m = A.mats + (size_t)matIdx * A.matStride + moff;
    if (child < 0) {
        const uint8_t* t = A.states + (size_t)(-child - 1) * A.Ppad;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int p = p0 + r * G;
            const bool active = catValid && p >= pBegin && p < pEnd;
            const int s = active ? (int)__ldg(t + p) : S;
            double v[4];
            if (s < S) ldg256_ro(m + 4 * CP * s, v);
            else {
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = (i < S) ? 1.0 : 0.0;
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) y[r][i] = FIRST ? v[i] : y[r][i] * v[i];
        }
    } else {
        Mat4 M;
        loadMat<CP>(m, M);
        const T* xg = static_cast<const T*>(A.partials) + (size_t)child * A.stride + off0;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int p = p0 + r * G;
            const bool active = catValid && p >= pBegin && p < pEnd;
            double x[4], v[4];
            if (STACK && slot != 0xFF) {
                double2 lo = stackMem[((slot * R + r) * 2 + 0) * nthreads + threadIdx.x];
                double2 hi = stackMem[((slot * R + r) * 2 + 1) * nthreads + threadIdx.x];
                x[0] = lo.x; x[1] = lo.y; x[2] = hi.x; x[3] = hi.y;
            } else if (active) {
                loadCell(xg + (size_t)r * G * 4, x);
            } else { x[0] = x[1] = x[2] = x[3] = 0.0; }
            applyMat(M, x, v);
#pragma unroll
            for (int i = 0; i < 4; ++i) y[r][i] = FIRST ? v[i] : y[r][i] * v[i];
        }
    }
}

template <typename T, int CP, int R, bool STACK, bool PRE>
__device__ __forceinline__ void walk4Body(const WalkArgs& A) {
    static_assert(sizeof(T) == 8 || !STACK, "the operand-stack variant is built for fp64 partials only");
    constexpr int G = 32 / CP;
    extern __shared__ double2 stackMem[];
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int c = lane / G;
    const int4 range = __ldg(A.subs + blockIdx.y);
    const int p0 = range.z + warp * (G * R) + (lane % G);          // patterns p0 + r*G
    if (range.z + warp * (G * R) >= range.w) return;               // whole warp outside this subtree's pattern window
    // (every op of a subtree carries the same [pBegin,pEnd) as the window, so the per-op range test suffices below)
    const bool catValid = c < A.C;
    const int cc = catValid ? c : 0;
    const size_t off0 = ((size_t)cc * A.Ppad + p0) * 4;
    const int moff = cc * 4;
    const int nthreads = blockDim.x;
    const int last = range.y - 1;

    Op4 cur = loadOp(A.ops + range.x);
    double d[R][4];                                            // survives the loop: op k+1 may take it as its first child
#pragma unroll
    for (int r = 0; r < R; ++r) d[r][0] = d[r][1] = d[r][2] = d[r][3] = 0.0;
    for (int k = range.x; k <= last; ++k) {
        // records: k+2 starts its trip to L1 now; k+1 is read (an L1 hit by then) only after this op's arithmetic, so
        // that its 16 registers are not live across the register-hungry part of the body
        // (R = 1, the latency-chain configuration, has registers to spare and reads k+1 a whole op ahead instead)
        Op4 nxt;
        if (R == 1) nxt = loadOp(A.ops + min(k + 1, last));
        else if (lane == 0) prefetchL1(A.ops + min(k + 2, last));
        const int s1 = cur.slots & 0xFF, s2 = (cur.slots >> 8) & 0xFF, sd = (cur.slots >> 16) & 0xFF;
        if (!STACK) {
            // look-ahead: the NEXT op's memory operands (never this op's destination) start their trip to L1 now,
            // so that its loads find them there when this op is done
#pragma unroll
            for (int w = 0; w < 2; ++w) {
                const int pf = w == 0 ? cur.pfA : cur.pfB;
                if (pf == 0) continue;
                if (pf & 1) {
                    const uint8_t* t = A.states + (size_t)(pf >> 1) * A.Ppad + p0;
                    if ((lane % G) == 0 && c == 0) prefetchL1(t);          // G*R consecutive bytes: one line
                } else if (catValid) {
                    const T* xg = static_cast<const T*>(A.partials) + (size_t)((pf >> 1) - 1) * A.stride + off0;
#pragma unroll
                    for (int r = 0; r < R; ++r)
                        if (p0 + r * G < A.Ppad) prefetchL1(xg + (size_t)r * G * 4);
                }
            }
            if (lane < 8) {
                const int mi = lane < 4 ? cur.pfM1 : cur.pfM2;
                if (mi >= 0) prefetchL1(A.mats + (size_t)mi * A.matStride + (lane & 3) * 4 * CP);
            }
        }
        if (!PRE) {
            if (!STACK && (cur.pad_ & 2)) {
                // the first child is what this very thread produced for the previous op of the walk: take it from
                // registers (no store -> L2 -> load round trip, one partial less through the LSU)
                Mat4 M;
                loadMat<CP>(A.mats + (size_t)cur.m1 * A.matStride + moff, M);
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    double v[4];
                    applyMat(M, d[r], v);
#pragma unroll
                    for (int i = 0; i < 4; ++i) d[r][i] = v[i];
                }
            } else {
                childTerm<T, CP, R, STACK, true>(A, cur.c1, cur.m1, s1, moff, off0, p0, catValid, cur.pBegin, cur.pEnd, stackMem, nthreads, d);
            }
            childTerm<T, CP, R, STACK, false>(A, cur.c2, cur.m2, s2, moff, off0, p0, catValid, cur.pBegin, cur.pEnd, stackMem, nthreads, d);
        } else {
            // pre-order op: q = pre[parent] (*) (M_sib post[sib]) at the parent, then down the node's own branch
            // with the transposed matrix: pre[node][j] = sum_i q[i] M_node[i][j]
            // (depth-first order inside a subtree walk: when this node is the first child of the previous op's node,
            // pre[parent] is still in d -- flag bit 1 -- and is not re-read)
            double v[R][4];
            childTerm<T, CP, R, false, true>(A, cur.c2, cur.m2, 0xFF, moff, off0, p0, catValid, cur.pBegin, cur.pEnd, stackMem, nthreads, v);
            Mat4 M1;
            loadMat<CP>(A.mats + (size_t)cur.m1 * A.matStride + moff, M1);
            const T* xg = static_cast<const T*>(A.partials) + (size_t)cur.c1 * A.stride + off0;
            const bool fromRegisters = (cur.pad_ & 2) != 0;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int p = p0 + r * G;
                double x[4] = {0.0, 0.0, 0.0, 0.0};
                if (fromRegisters) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) x[i] = d[r][i];
                } else if (catValid && p >= cur.pBegin && p < cur.pEnd) loadCell(xg + (size_t)r * G * 4, x);
                double q[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) q[i] = x[i] * v[r][i];
#pragma unroll
                for (int j = 0; j < 4; ++j) d[r][j] = M1.r[j][0] * q[0] + M1.r[j][1] * q[1] + M1.r[j][2] * q[2] + M1.r[j][3] * q[3];
            }
        }
        if (R != 1) nxt = loadOp(A.ops + min(k + 1, last));
        T* dg = static_cast<T*>(A.partials) + (size_t)cur.dest * A.stride + off0;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int p = p0 + r * G;
            const bool active = catValid && p >= cur.pBegin && p < cur.pEnd;
            // ---- rescaling (AbstractLikelihoodCore.java:406-442, unconditional as in BEAGLE) -----
            if (cur.sw >= 0) {
                double m = active ? fmax(fmax(d[r][0], d[r][1]), fmax(d[r][2], d[r][3])) : 0.0;
#pragma unroll
                for (int sh = G; sh < 32; sh <<= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, sh));
                if (m == 0.0) m = 1.0;
                const double inv = 1.0 / m;
#pragma unroll
                for (int i = 0; i < 4; ++i) d[r][i] *= inv;
                if (active && c == 0) {
                    // raw scalers need no logarithm here; cumulative buffers are accumulated by k_scale_accum after the
                    // phases (an in-walk "cum += log m" would race between concurrent subtrees)
                    A.scale[(size_t)cur.sw * A.Ppad + p] = A.logScalers ? log(m) : m;
                }
                __syncwarp();
            } else if (cur.sr >= 0) {
                double f = active ? A.scale[(size_t)cur.sr * A.Ppad + p] : 1.0;
                if (A.logScalers) f = exp(f);
                const double inv = 1.0 / f;
#pragma unroll
                for (int i = 0; i < 4; ++i) d[r][i] *= inv;
            }
            roundCell<T>(d[r]);
            if (active) storeCell(dg + (size_t)r * G * 4, d[r]);
            if (STACK && sd != 0xFF) {
                stackMem[((sd * R + r) * 2 + 0) * nthreads + threadIdx.x] = make_double2(d[r][0], d[r][1]);
                stackMem[((sd * R + r) * 2 + 1) * nthreads + threadIdx.x] = make_double2(d[r][2], d[r][3]);
            }
        }
        cur = nxt;
    }
}

template <int CP, int R, bool STACK, int MINB, bool PRE>
__global__ void __launch_bounds__(128, MINB)
k_walk4(const WalkArgs A) {
    walk4Body<double, CP, R, STACK, PRE>(A);
}

// fp32 partials storage (PRECISION_SINGLE); no operand-stack variant
template <int CP, int R, int MINB, bool PRE>
__global__ void __launch_bounds__(128, MINB)
k_walk4s(const WalkArgs A) {
    walk4Body<float, CP, R, false, PRE>(A);
}

template <int CP, int R, bool STACK, int MINB, bool PRE = false>
static cudaError_t launchWalk4K(Instance* in, const WalkArgs& A, dim3 grid, size_t smem) {
    if (in->single) {                  // the stack variant never runs on a single instance (walkVariant = stackTail = 0)
        if constexpr (!STACK && CP <= 8) k_walk4s<CP, R, MINB, PRE><<<grid, 128, 0, in->stream>>>(A);
        else return cudaErrorInvalidValue;
        return cudaGetLastError();
    }
    if (smem > 0 && smem > in->walkSmemConfigured) {
        cudaError_t e = cudaFuncSetAttribute(k_walk4<CP, R, STACK, MINB, PRE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        in->walkSmemConfigured = smem;
    }
    k_walk4<CP, R, STACK, MINB, PRE><<<grid, 128, smem, in->stream>>>(A);
    return cudaGetLastError();
}

template <int CP, int R>
static cudaError_t launchWalk4R(Instance* in, const Op4* dOps, const int4* dSubs, int nSubs, int stackDepth, int maxWindow, bool preOrder) {
    constexpr int G = 32 / CP;
    const int warps = (maxWindow + G * R - 1) / (G * R);
    dim3 grid((warps + 3) / 4, nSubs);
    WalkArgs A;
    A.ops = dOps; A.subs = dSubs; A.partials = in->partialsBase; A.stride = in->partialsElems;
    A.states = in->states8Base; A.mats = in->dMat; A.scale = in->dScale;
    A.S = in->S; A.C = in->C; A.Ppad = in->Ppad; A.logScalers = in->logScalers ? 1 : 0;
    A.matStride = in->matStride; A.matMmaOffset = 16 * in->matCP;
    if (preOrder) return launchWalk4K<CP, R, false, 4, true>(in, A, grid, 0);
    if (stackDepth > 0) return launchWalk4K<CP, R, true, 4>(in, A, grid, (size_t)stackDepth * 32 * R * 128);
    if (in->walkMinBlocks >= 6) return launchWalk4K<CP, R, false, 6>(in, A, grid, 0);
    if (in->walkMinBlocks == 5) return launchWalk4K<CP, R, false, 5>(in, A, grid, 0);
    if (in->walkMinBlocks == 3) return launchWalk4K<CP, R, false, 3>(in, A, grid, 0);
    return launchWalk4K<CP, R, false, 4>(in, A, grid, 0);
}

// ---------------------------------------------------------------------------------------------
// 4-state walk on the FP64 tensor pipe (DMMA m8n8k4)  --  B200_WALK_VARIANT=2
// ---------------------------------------------------------------------------------------------
// D[p][i] = sum_j X[p][j] * P[i][j]  as one mma.sync.m8n8k4.f64 per (8 patterns, category, child):
//   A fragment = child partials  [8 patterns][4 states]   lane (g,t) <- X[p0+g][t]     (256 contiguous bytes / warp)
//   B fragment = transition rows [4 (j)][8 (i)]            lane (g,t) <- Mpad[g][t]     (256 contiguous bytes, rows >= 4 zero)
//   D fragment                    [8 patterns][8 (i)]      lane (g,t) -> i = 2t,2t+1 of pattern g (meaningful for t < 2)
// wgmma has no fp64 kind, so the fp64 tensor path on sm_90a is mma.sync (SASS DMMA.8x8x4).
// The matrix reaches the register file ONCE per warp (8 B/lane) instead of once per thread (128 B/lane),
// which is what saturates the LSU->RF path of the FMA kernel.  Everything is arranged so that loads need
// no predicates: pattern rows are padded to 32, gap tips read a ones-column, B rows 4..7 are stored zeros;
// only stores (and scale-factor writes) are masked.  Warp = C categories x R tiles of 8 patterns.
__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%4,%5};"
        : "=d"(d0), "=d"(d1) : "d"(a), "d"(b), "d"(0.0), "d"(0.0));
}

template <int C, int R, int MINB>
__global__ void __launch_bounds__(128, MINB)
k_walk4t(const WalkArgs A) {
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int4 range = __ldg(A.subs + blockIdx.y);
    if (range.z + warp * (8 * R) >= range.w) return;
    const int g = lane >> 2, t = lane & 3;
    const int pBase = range.z + warp * (8 * R) + g;        // pattern of tile r: pBase + 8 r   (always < Ppad)
    const size_t mstride = A.matStride;
    const size_t catStride = (size_t)A.Ppad * 4;
    const size_t cellOff = (size_t)pBase * 4;
    const int last = range.y - 1;
    const double* matB = A.mats + A.matMmaOffset + lane;                    // Mpad[c][g][t] = + c*32
    const double* matT = A.mats + A.matMmaOffset + C * 32 + 2 * (t & 1);     // MTg[c][s][2t..] = + c*20 + s*4

    Op4 cur = loadOp(A.ops + range.x);
    for (int k = range.x; k <= last; ++k) {
        const Op4 nxt = loadOp(A.ops + min(k + 1, last));
        double y[C][R][2];
#pragma unroll
        for (int child = 0; child < 2; ++child) {
            const int cb = child == 0 ? cur.c1 : cur.c2;
            const size_t moff = (size_t)(child == 0 ? cur.m1 : cur.m2) * mstride;
            if (cb >= 0) {
                const double* x = static_cast<const double*>(A.partials) + (size_t)cb * A.stride + cellOff + t;
                double b[C];
#pragma unroll
                for (int c = 0; c < C; ++c) b[c] = __ldg(matB + moff + c * 32);
#pragma unroll
                for (int c = 0; c < C; ++c) {
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        double a, d0, d1;
                        asm volatile("ld.global.f64 %0, [%1];" : "=d"(a) : "l"(x + c * catStride + r * 32) : "memory");
                        dmma884(d0, d1, a, b[c]);
                        if (child == 0) { y[c][r][0] = d0; y[c][r][1] = d1; }
                        else { y[c][r][0] *= d0; y[c][r][1] *= d1; }
                    }
                }
            } else {
                const uint8_t* st = A.states + (size_t)(-cb - 1) * A.Ppad + pBase;
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const int s = (int)__ldg(st + 8 * r);                    // gap/unknown is stored as S -> ones column
                    const double* col = matT + moff + s * 4;
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        const double2 v = __ldg(reinterpret_cast<const double2*>(col + c * 20));
                        if (child == 0) { y[c][r][0] = v.x; y[c][r][1] = v.y; }
                        else { y[c][r][0] *= v.x; y[c][r][1] *= v.y; }
                    }
                }
            }
        }
        // ---- fused rescale (AbstractLikelihoodCore.java:406-442, unconditional as in BEAGLE) ---------
        if (cur.sw >= 0 || cur.sr >= 0) {
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int p = pBase + 8 * r;
                const bool act = p >= cur.pBegin && p < cur.pEnd;
                double f;
                if (cur.sw >= 0) {
                    double m = 0.0;
#pragma unroll
                    for (int c = 0; c < C; ++c) m = fmax(m, fmax(y[c][r][0], y[c][r][1]));
                    if (t >= 2) m = 0.0;                                     // lanes t >= 2 carry no states
                    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 1));
                    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 2));
                    if (m == 0.0) m = 1.0;
                    f = m;
                    if (act && t == 0) {
                        A.scale[(size_t)cur.sw * A.Ppad + p] = A.logScalers ? log(m) : m;
                    }
                } else {
                    f = act ? A.scale[(size_t)cur.sr * A.Ppad + p] : 1.0;
                    if (A.logScalers) f = exp(f);
                }
                const double inv = 1.0 / f;
#pragma unroll
                for (int c = 0; c < C; ++c) { y[c][r][0] *= inv; y[c][r][1] *= inv; }
            }
        }
        // ---- store: lanes t < 2 own states 2t, 2t+1 (16 B) of pattern g ---------------------------
        {
            double* dst = static_cast<double*>(A.partials) + (size_t)cur.dest * A.stride + cellOff + 2 * t;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int p = pBase + 8 * r;
                if (t < 2 && p >= cur.pBegin && p < cur.pEnd) {
#pragma unroll
                    for (int c = 0; c < C; ++c)
                        asm volatile("st.global.v2.f64 [%0], {%1,%2};" :: "l"(dst + c * catStride + r * 32),
                                     "d"(y[c][r][0]), "d"(y[c][r][1]) : "memory");
                }
            }
        }
        __syncwarp();          // the next op may read (through other lanes of this warp) what was just stored
        cur = nxt;
    }
}

template <int C, int R>
static cudaError_t launchWalk4Tensor(Instance* in, const Op4* dOps, const int4* dSubs, int nSubs, int maxWindow) {
    const int warps = (maxWindow + 8 * R - 1) / (8 * R);
    dim3 grid((warps + 3) / 4, nSubs);
    WalkArgs A;
    A.ops = dOps; A.subs = dSubs; A.partials = in->partialsBase; A.stride = in->partialsElems;
    A.states = in->states8Base; A.mats = in->dMat; A.scale = in->dScale;
    A.S = in->S; A.C = in->C; A.Ppad = in->Ppad; A.logScalers = in->logScalers ? 1 : 0;
    A.matStride = in->matStride; A.matMmaOffset = 16 * in->matCP;
    if (in->walkMinBlocks >= 6) k_walk4t<C, R, 6><<<grid, 128, 0, in->stream>>>(A);
    else k_walk4t<C, R, 4><<<grid, 128, 0, in->stream>>>(A);
    return cudaGetLastError();
}

// exact category counts only (fully unrolled); anything else stays on the FMA kernel
static bool walk4TensorSupported(const Instance* in) { return in->C == 1 || in->C == 2 || in->C == 4 || in->C == 8; }

static cudaError_t launchWalk4Mma(Instance* in, const Op4* dOps, const int4* dSubs, int nSubs, int maxWindow) {
    const bool r4 = in->tensorR >= 4;
    switch (in->C) {
        case 1: return r4 ? launchWalk4Tensor<1, 4>(in, dOps, dSubs, nSubs, maxWindow) : launchWalk4Tensor<1, 2>(in, dOps, dSubs, nSubs, maxWindow);
        case 2: return r4 ? launchWalk4Tensor<2, 4>(in, dOps, dSubs, nSubs, maxWindow) : launchWalk4Tensor<2, 2>(in, dOps, dSubs, nSubs, maxWindow);
        case 4: return r4 ? launchWalk4Tensor<4, 4>(in, dOps, dSubs, nSubs, maxWindow) : launchWalk4Tensor<4, 2>(in, dOps, dSubs, nSubs, maxWindow);
        default: return launchWalk4Tensor<8, 2>(in, dOps, dSubs, nSubs, maxWindow);
    }
}

template <int CP>
static cudaError_t launchWalk4T(Instance* in, const Op4* dOps, const int4* dSubs, int nSubs, int stackDepth, int maxWindow, bool preOrder) {
    // a thin phase (few walks in flight) is latency-bound: one pattern group per thread gives 4x the warps per op
    const long walks = (long)nSubs * ((maxWindow + (32 / CP) * in->walkR - 1) / ((32 / CP) * in->walkR));
    if (in->thinR1 && stackDepth == 0 && walks < (long)in->smCount * 8)
        return launchWalk4R<CP, 1>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
    switch (in->walkR) {
        case 4: return launchWalk4R<CP, 4>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
        case 2: return launchWalk4R<CP, 2>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
        default: return launchWalk4R<CP, 1>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
    }
}

cudaError_t launchWalk4(Instance* in, const Op4* dOps, const int4* dSubs, int nSubs, int stackDepth, int maxWindow, bool preOrder) {
    if (nSubs <= 0) return cudaSuccess;
    if (in->walkVariant == 2 && !preOrder && walk4TensorSupported(in)) return launchWalk4Mma(in, dOps, dSubs, nSubs, maxWindow);
    switch (in->matCP) {
        case 1: return launchWalk4T<1>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
        case 2: return launchWalk4T<2>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
        case 4: return launchWalk4T<4>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
        case 8: return launchWalk4T<8>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
        case 16: return launchWalk4T<16>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
        default: return launchWalk4T<32>(in, dOps, dSubs, nSubs, stackDepth, maxWindow, preOrder);
    }
}

// ---------------------------------------------------------------------------------------------
// generic-state block walk
// ---------------------------------------------------------------------------------------------
// Block owns TP consecutive patterns and walks the op list; per (op, category) it stages the two
// transposed matrices and the two child tiles in shared memory, computes the TP x Sp destination
// tile (thread index = pattern-major, parent state fastest: conflict-free matrix reads, broadcast
// child reads, coalesced stores), tracks per-pattern maxima for the optional rescale.
__global__ void __launch_bounds__(256)
k_walk_generic(const DevOp* __restrict__ ops, const int4* __restrict__ subs, int S, int Sp, int C, int Ppad, int TP,
               int logScalers, int stageMatrices, int hasPre) {
    extern __shared__ double smg[];
    const size_t msz = stageMatrices ? (size_t)Sp * Sp : 0;
    double* mt1s = smg;
    double* mt2s = smg + msz;
    double* x1 = smg + 2 * msz;
    double* x2 = x1 + (size_t)TP * Sp;
    double* qt = x2 + (size_t)TP * Sp;                       // pre-order lists only: q tile
    unsigned long long* pmax = reinterpret_cast<unsigned long long*>(qt + (hasPre ? (size_t)TP * Sp : 0));
    const int4 range = subs[blockIdx.y];
    const int p0 = range.z + blockIdx.x * TP;
    if (p0 >= range.w) return;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int tileElems = min(TP, Ppad - p0) * Sp;          // never read past the slab's last pattern

    for (int k = range.x; k < range.y; ++k) {
        const DevOp op = ops[k];
        const bool doMax = op.scaleWrite != nullptr;
        if (doMax) for (int q = tid; q < TP; q += nt) pmax[q] = 0ull;
        for (int c = 0; c < C; ++c) {
            __syncthreads();
            const bool pre = (op.pad_ & 1) != 0;
            // pre-order ops use the ROW-MAJOR copy of the node's own matrix (second half of the buffer)
            const int ld1 = pre ? Sp + 4 : Sp;       // the row-major copy carries the tensor path's padded row stride
            const double* m1g = op.m1 + (pre ? (size_t)C * Sp * Sp + (size_t)c * Sp * ld1 : (size_t)c * Sp * Sp);
            const double* m2g = op.m2 + (size_t)c * Sp * Sp;
            if (stageMatrices) {
                for (int q = tid; q < Sp * Sp; q += nt) { mt1s[q] = m1g[(q / Sp) * ld1 + (q % Sp)]; mt2s[q] = m2g[q]; }
            }
            const size_t tileOff = ((size_t)c * Ppad + p0) * Sp;
            if (op.c1) for (int q = tid; q < tileElems; q += nt) x1[q] = op.c1[tileOff + q];
            if (op.c2) for (int q = tid; q < tileElems; q += nt) x2[q] = op.c2[tileOff + q];
            __syncthreads();
            const double* mt1 = stageMatrices ? mt1s : m1g;
            const double* mt2 = stageMatrices ? mt2s : m2g;
            if (pre) {
                // stage A: q[i] = pre[parent][i] * (M_sib post[sib])[i]
                for (int q = tid; q < tileElems; q += nt) {
                    const int pl = q / Sp, i = q - pl * Sp;
                    const int p = p0 + pl;
                    double b = 0.0;
                    if (p >= op.pBegin && p < op.pEnd && p < range.w) {
                        if (op.c2) {
                            const double* xr = x2 + (size_t)pl * Sp;
                            for (int j = 0; j < S; ++j) b += mt2[(size_t)j * Sp + i] * xr[j];
                        } else {
                            int s = static_cast<const int*>(op.s2)[p];
                            b = (s < S) ? mt2[(size_t)s * Sp + i] : ((i < S) ? 1.0 : 0.0);
                        }
                        b *= x1[q];
                    }
                    qt[q] = b;
                }
                __syncthreads();
                // stage B: pre[node][j] = sum_i q[i] M_node[i][j]   (row-major matrix: conflict-free in j)
                for (int q = tid; q < tileElems; q += nt) {
                    const int pl = q / Sp, j = q - pl * Sp;
                    const int p = p0 + pl;
                    if (!(p >= op.pBegin && p < op.pEnd && p < range.w)) continue;
                    double d = 0.0;
                    const double* qr = qt + (size_t)pl * Sp;
                    for (int i = 0; i < S; ++i) d += qr[i] * mt1[(size_t)i * (stageMatrices ? Sp : ld1) + j];
                    op.dest[tileOff + q] = d;
                    if (doMax) atomicMax(&pmax[pl], (unsigned long long)__double_as_longlong(d));
                }
                continue;
            }
            for (int q = tid; q < tileElems; q += nt) {
                const int pl = q / Sp, i = q - pl * Sp;
                const int p = p0 + pl;
                const bool active = p >= op.pBegin && p < op.pEnd && p < range.w;
                if (!active) continue;
                double a, b;
                if (op.c1) {
                    a = 0.0;
                    const double* xr = x1 + (size_t)pl * Sp;
                    for (int j = 0; j < S; ++j) a += mt1[(size_t)j * Sp + i] * xr[j];
                } else {
                    int s = static_cast<const int*>(op.s1)[p];
                    a = (s < S) ? mt1[(size_t)s * Sp + i] : ((i < S) ? 1.0 : 0.0);
                }
                if (op.c2) {
                    b = 0.0;
                    const double* xr = x2 + (size_t)pl * Sp;
                    for (int j = 0; j < S; ++j) b += mt2[(size_t)j * Sp + i] * xr[j];
                } else {
                    int s = static_cast<const int*>(op.s2)[p];
                    b = (s < S) ? mt2[(size_t)s * Sp + i] : ((i < S) ? 1.0 : 0.0);
                }
                const double d = a * b;
                op.dest[tileOff + q] = d;
                if (doMax) atomicMax(&pmax[pl], (unsigned long long)__double_as_longlong(d));
            }
        }
        if (op.scaleWrite != nullptr || op.scaleRead != nullptr) {
            __syncthreads();
            for (int c = 0; c < C; ++c) {
                const size_t tileOff = ((size_t)c * Ppad + p0) * Sp;
                for (int q = tid; q < tileElems; q += nt) {
                    const int pl = q / Sp;
                    const int p = p0 + pl;
                    if (p < op.pBegin || p >= op.pEnd || p >= range.w) continue;
                    double f;
                    if (op.scaleWrite) {
                        f = __longlong_as_double((long long)pmax[pl]);
                        if (f == 0.0) f = 1.0;
                    } else {
                        f = op.scaleRead[p];
                        if (logScalers) f = exp(f);
                    }
                    op.dest[tileOff + q] *= (1.0 / f);
                }
            }
            if (op.scaleWrite) {
                for (int pl = tid; pl < TP; pl += nt) {
                    const int p = p0 + pl;
                    if (p < op.pBegin || p >= op.pEnd || p >= range.w) continue;
                    double m = __longlong_as_double((long long)pmax[pl]);
                    if (m == 0.0) m = 1.0;
                    op.scaleWrite[p] = logScalers ? log(m) : m;
                }
            }
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------------------------------------
// generic-state block walk on the FP64 tensor pipe (DMMA m8n8k4): amino-acid (20) and codon (61) models
// ---------------------------------------------------------------------------------------------
// Per (op, category) the contraction D[p][i] = sum_j X[p][j] P[i][j] is a (patterns x Sp) * (Sp x Sp)
// GEMM: A fragments come straight from the child partials in global memory (each element is read
// exactly once per op, so there is nothing to stage), B fragments from the row-major matrix staged in
// shared memory with a (Sp+4)-double row stride (conflict-free for the 8x4 fragment shape), and the
// 16 x Sp accumulator tile of each warp lives in registers.  Block = 4 warps x 16 patterns.

__device__ __forceinline__ void cpAsync16(void* smemDst, const void* gmemSrc) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smemDst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s), "l"(gmemSrc) : "memory");
}

// x where `on`, else 0, as one selp the compiler cannot see through: a plain `on ? x : 0.0` ahead of an mma.sync lets it
// specialise the mma per lane (zero operands folded, predicated copies), and mma.sync.aligned on diverged lanes deadlocks
__device__ __forceinline__ double selOn(double x, bool on) {
    double r;
    asm volatile("{\n.reg .pred p;\nsetp.ne.u32 p, %2, 0;\nselp.f64 %0, %1, 0d0000000000000000, p;\n}\n"
                 : "=d"(r) : "d"(x), "r"((unsigned)on));
    return r;
}

// ---- TMA (1-D bulk copy) staging: one elected thread moves a whole padded matrix, completion on an mbarrier ----
__device__ __forceinline__ void mbarInit(uint64_t* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbarExpectTx(uint64_t* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarWait(uint64_t* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" :: "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulkCopyG2S(void* smemDst, const void* gmemSrc, unsigned bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"((unsigned)__cvta_generic_to_shared(smemDst)), "l"(gmemSrc), "r"(bytes),
                    "r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
}

// Block = WARPS warps x 16 patterns.  Per (op, category) ONE thread issues two bulk copies (TMA engine, SASS UBLKCP):
// the matrices sit in global memory already in the padded [Sp][Sp+4] shape the fragment loads want, so each is one
// contiguous transfer; everyone else waits on the mbarrier and spends no issue slots on staging.  Single buffer: the
// other resident blocks of the SM cover the copy (measured faster than a double buffer at one block per SM).
// MT = 8-pattern m-tiles per warp: 2 where the launch fills the GPU (each B fragment feeds two DMMAs), 1 for the thin phases near
// the root, where twice as many (half as tall) blocks put every SM to work
template <int NT, int WARPS, bool PRE, bool MULTI, int MT = 2>
__global__ void __launch_bounds__(WARPS * 32, 3)
k_walk_mma(const DevOp* __restrict__ ops, const int4* __restrict__ subs, int S, int C, int Ppad, int logScalers, int cbArg) {
    static_assert(MT == 2 || (MT == 1 && !PRE), "the pre-order form keeps two m-tiles per warp");
    const int cb = MULTI ? cbArg : 1;               // MULTI = false: one category per staging round, folded at compile time
    constexpr int Sp = 8 * NT;
    constexpr int LD = Sp + 4;                       // shared-memory row stride (doubles)
    constexpr int MATSZ = Sp * LD;
    constexpr unsigned MATBYTES = MATSZ * sizeof(double);
    // [child 1: cb categories][child 2: cb categories] x [Sp][LD]; cb = categories staged per bulk copy (small state
    // counts stage all of an op's categories at once: one barrier round trip per op instead of one per category)
    extern __shared__ __align__(128) double smw[];
    __shared__ __align__(8) uint64_t bar;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int4 range = subs[blockIdx.y];
    if (range.z + blockIdx.x * (WARPS * 8 * MT) >= range.w) return;  // block outside this subtree's pattern window
    const int pw = range.z + blockIdx.x * (WARPS * 8 * MT) + w * 8 * MT;   // first pattern of this warp's (8 MT)-row tile
    const size_t mRow = (size_t)C * Sp * Sp;         // offset of the padded row-major copies in a matrix buffer
    const size_t mTp = mRow + (size_t)C * MATSZ;     // offset of the padded transposed copies
    const int total = (range.y - range.x) * C;
    if (tid == 0) {
        mbarInit(&bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    unsigned parity = 0;

    bool act[MT];
    double rowMax[MT];
#pragma unroll
    for (int m = 0; m < MT; ++m) { act[m] = false; rowMax[m] = 0.0; }
    // the accumulator tile outlives the iteration: with one category the next op of the walk may take it as its first
    // child straight from these registers (DevOp::pad_ bit 1, set by the planner as for the 4-state walk)
    double acc[MT][NT][2];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int n = 0; n < NT; ++n) { acc[m][n][0] = 0.0; acc[m][n][1] = 0.0; }
    for (int flat = 0; flat < total; ++flat) {
        const int c = flat % C, cg = c % cb;
        if (cg == 0) {
            if (tid == 0) {
                const DevOp* o = ops + range.x + flat / C;
                const unsigned bytes = (unsigned)min(cb, C - c) * MATBYTES;       // consecutive categories are contiguous
                // pre-order ops contract over the ROW index of the node's own matrix: stage its transposed copy
                // a compact-tip child of a post-order op only needs COLUMN s of its matrix: stage the transposed copy, where
                // that column is one contiguous row (two LDS.128 per accumulator pair instead of bank-conflicting LDS.64s)
                const double* g1 = o->m1 + ((PRE || o->c1 == nullptr) ? mTp : mRow) + (size_t)c * MATSZ;
                const double* g2 = o->m2 + ((!PRE && o->c2 == nullptr) ? mTp : mRow) + (size_t)c * MATSZ;
                // the generic-proxy reads of the previous group (ordered by the barrier that ended it) precede these writes
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                mbarExpectTx(&bar, 2 * bytes);
                bulkCopyG2S(smw, g1, bytes, &bar);
                bulkCopyG2S(smw + (size_t)cb * MATSZ, g2, bytes, &bar);
            }
            mbarWait(&bar, parity);
            parity ^= 1;
        }
        const DevOp op = ops[range.x + flat / C];
        const double* P1 = smw + (size_t)cg * MATSZ;
        const double* P2 = smw + (size_t)(cb + cg) * MATSZ;
        if (c == 0) {
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                const int p = pw + 8 * m + g;
                act[m] = p < range.w && p >= op.pBegin && p < op.pEnd;
                rowMax[m] = 0.0;
            }
        }
        if constexpr (PRE) {
            // pre[node][j] = sum_i ( pre[parent][i] * (M_sib post[sib])[i] ) M_node[i][j]
            // (1) v = M_sib post[sib] on the tensor pipe (or a column lookup for a compact tip)
            double u[2][NT][2];
            if (op.c2 != nullptr) {
#pragma unroll
                for (int m = 0; m < 2; ++m)
#pragma unroll
                    for (int n = 0; n < NT; ++n) { u[m][n][0] = 0.0; u[m][n][1] = 0.0; }
                // mma.sync is .aligned: every lane must reach it on the same path.  Guarded loads let the compiler branch
                // per lane (and deadlock a warp whose patterns straddle the end of the window), so every lane loads from
                // a row clamped into the padded buffer and inactive lanes select zero (selOn).
                const double* xrow0 = op.c2 + ((size_t)c * Ppad + min(pw + g, Ppad - 1)) * Sp + t;
                const double* xrow1 = op.c2 + ((size_t)c * Ppad + min(pw + 8 + g, Ppad - 1)) * Sp + t;
                const double* brow = P2 + g * LD + t;
#pragma unroll 4
                for (int kc = 0; kc < Sp / 4; ++kc) {
                    const double x0 = xrow0[4 * kc], x1 = xrow1[4 * kc];
                    const double a0 = selOn(x0, act[0]), a1 = selOn(x1, act[1]);
#pragma unroll
                    for (int n = 0; n < NT; ++n) {
                        const double b = brow[n * 8 * LD + 4 * kc];
                        dmma884acc(u[0][n][0], u[0][n][1], a0, b);
                        dmma884acc(u[1][n][0], u[1][n][1], a1, b);
                    }
                }
            } else {
                const int* st = static_cast<const int*>(op.s2);
#pragma unroll
                for (int m = 0; m < 2; ++m) {
                    const int s = act[m] ? st[pw + 8 * m + g] : S;
#pragma unroll
                    for (int n = 0; n < NT; ++n)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int i = 8 * n + 2 * t + e;
                            u[m][n][e] = (s < S) ? P2[i * LD + s] : ((i < S) ? 1.0 : 0.0);
                        }
                }
            }
            // (2) times the parent's pre-order partial, read in the accumulator layout
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                const double* prow = op.c1 + ((size_t)c * Ppad + (pw + 8 * m + g)) * Sp + 2 * t;
#pragma unroll
                for (int n = 0; n < NT; ++n) {
                    double2 v = make_double2(0.0, 0.0);
                    if (act[m]) v = *reinterpret_cast<const double2*>(prow + 8 * n);
                    u[m][n][0] *= v.x; u[m][n][1] *= v.y;
                    acc[m][n][0] = 0.0; acc[m][n][1] = 0.0;
                }
            }
            // (3) second contraction.  The sum over i may visit the states in any order, so k-chunk (n, e0) is
            // DEFINED as the four states lane t already holds: i = 8n + 2t + (e0 ^ (t >> 1)) -- no accumulator ->
            // A-fragment shuffle, and with the (Sp+4) row stride the B reads stay bank-conflict free.
            const int flip = t >> 1;
            const double* brow = P1 + g * LD + 2 * t;
#pragma unroll
            for (int n = 0; n < NT; ++n)
#pragma unroll
                for (int e0 = 0; e0 < 2; ++e0) {
                    const int e = e0 ^ flip;
                    const double a0 = e ? u[0][n][1] : u[0][n][0];
                    const double a1 = e ? u[1][n][1] : u[1][n][0];
#pragma unroll
                    for (int n2 = 0; n2 < NT; ++n2) {
                        const double b = brow[n2 * 8 * LD + 8 * n + e];
                        dmma884acc(acc[0][n2][0], acc[0][n2][1], a0, b);
                        dmma884acc(acc[1][n2][0], acc[1][n2][1], a1, b);
                    }
                }
        } else {
#pragma unroll
        for (int child = 0; child < 2; ++child) {
            const double* xg = child == 0 ? op.c1 : op.c2;
            const double* Ps = child == 0 ? P1 : P2;
            double cur[MT][NT][2];
            if (xg != nullptr) {
#pragma unroll
                for (int m = 0; m < MT; ++m)
#pragma unroll
                    for (int n = 0; n < NT; ++n) { cur[m][n][0] = 0.0; cur[m][n][1] = 0.0; }
                // The sum over the child's states j may visit them in any order, so k-chunk (n, e0) is DEFINED as the four
                // states the lanes t = 0..3 hold in the ACCUMULATOR layout: j = 8n + 2t + (e0 ^ (t >> 1)).  The child tile is
                // then read exactly as it was written (one 16-byte load per lane and state pair, half the instructions of the
                // fragment-shaped 8-byte loads) -- or not read at all: when the child is the previous op's result, the
                // A operands ARE the accumulator registers (no shuffle, no memory), with the same arithmetic either way.
                const bool fwd = child == 0 && C == 1 && (op.pad_ & 2) != 0;
                const int flip = t >> 1;
                const double* xrow = xg + ((size_t)c * Ppad + (pw + g)) * Sp + 2 * t;      // m-tile m: + m * 8 rows
                const double* brow = Ps + g * LD + 2 * t;
                bool ld[MT];
                double2 x[MT];
#pragma unroll
                for (int m = 0; m < MT; ++m) {
                    ld[m] = act[m] && !fwd;
                    x[m] = make_double2(0.0, 0.0);
                    if (ld[m]) x[m] = *reinterpret_cast<const double2*>(xrow + (size_t)m * 8 * Sp);
                }
#pragma unroll
                for (int n = 0; n < NT; ++n) {
                    double2 nx[MT];
                    double v[MT][2];
#pragma unroll
                    for (int m = 0; m < MT; ++m) {
                        nx[m] = make_double2(0.0, 0.0);                     // the next state pair travels while this one computes
                        if (n + 1 < NT && ld[m]) nx[m] = *reinterpret_cast<const double2*>(xrow + (size_t)m * 8 * Sp + 8 * (n + 1));
                        v[m][0] = fwd ? acc[m][n][0] : x[m].x;
                        v[m][1] = fwd ? acc[m][n][1] : x[m].y;
                    }
#pragma unroll
                    for (int e0 = 0; e0 < 2; ++e0) {
                        const int e = e0 ^ flip;
                        double a[MT];
#pragma unroll
                        for (int m = 0; m < MT; ++m) a[m] = e ? v[m][1] : v[m][0];
#pragma unroll
                        for (int n2 = 0; n2 < NT; ++n2) {
                            const double b = brow[n2 * 8 * LD + 8 * n + e];
#pragma unroll
                            for (int m = 0; m < MT; ++m) dmma884acc(cur[m][n2][0], cur[m][n2][1], a[m], b);
                        }
                    }
#pragma unroll
                    for (int m = 0; m < MT; ++m) x[m] = nx[m];
                }
            } else {
                const int* st = static_cast<const int*>(child == 0 ? op.s1 : op.s2);
#pragma unroll
                for (int m = 0; m < MT; ++m) {
                    const int p = pw + 8 * m + g;
                    const int s = act[m] ? st[p] : S;
                    const double* col = Ps + (size_t)(s < S ? s : 0) * LD + 2 * t;      // staged TRANSPOSED: row s = column s of P
#pragma unroll
                    for (int n = 0; n < NT; ++n) {
                        const double2 v = *reinterpret_cast<const double2*>(col + 8 * n);
                        cur[m][n][0] = (s < S) ? v.x : ((8 * n + 2 * t < S) ? 1.0 : 0.0);
                        cur[m][n][1] = (s < S) ? v.y : ((8 * n + 2 * t + 1 < S) ? 1.0 : 0.0);
                    }
                }
            }
#pragma unroll
            for (int m = 0; m < MT; ++m)
#pragma unroll
                for (int n = 0; n < NT; ++n)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        acc[m][n][e] = child == 0 ? cur[m][n][e] : acc[m][n][e] * cur[m][n][e];
        }
        }
        // one category (the codon workloads): the per-pattern factor is known before anything is stored -- scale the
        // accumulators in registers and write the tile ONCE (the general path below re-reads and re-writes C tiles)
        const bool scaleInRegisters = C == 1 && (op.scaleWrite != nullptr || op.scaleRead != nullptr);
        if (scaleInRegisters) {
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                const int p = pw + 8 * m + g;
                double f;
                if (op.scaleWrite != nullptr) {
                    double mx = 0.0;
#pragma unroll
                    for (int n = 0; n < NT; ++n) mx = fmax(mx, fmax(acc[m][n][0], acc[m][n][1]));
                    if (!act[m]) mx = 0.0;
                    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    if (mx == 0.0) mx = 1.0;
                    f = mx;
                    if (act[m] && t == 0) op.scaleWrite[p] = logScalers ? log(mx) : mx;
                } else {
                    f = act[m] ? op.scaleRead[p] : 1.0;
                    if (logScalers) f = exp(f);
                }
                const double inv = 1.0 / f;
#pragma unroll
                for (int n = 0; n < NT; ++n) { acc[m][n][0] *= inv; acc[m][n][1] *= inv; }
            }
        }
        // store the tile: lane (g,t) owns states 8n+2t, 8n+2t+1 of rows g and g+8
#pragma unroll
        for (int m = 0; m < MT; ++m) {
            if (!act[m]) continue;
            double* drow = op.dest + ((size_t)c * Ppad + (pw + 8 * m + g)) * Sp + 2 * t;
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                *reinterpret_cast<double2*>(drow + 8 * n) = make_double2(acc[m][n][0], acc[m][n][1]);
                rowMax[m] = fmax(rowMax[m], fmax(acc[m][n][0], acc[m][n][1]));
            }
        }
        if (c == C - 1 && !scaleInRegisters && (op.scaleWrite != nullptr || op.scaleRead != nullptr)) {
            // per-pattern factor (max over categories and states), then one more pass over what this
            // warp just wrote (same lanes re-read their own stores)
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                const int p = pw + 8 * m + g;
                double f;
                if (op.scaleWrite != nullptr) {
                    double mx = act[m] ? rowMax[m] : 0.0;
                    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    if (mx == 0.0) mx = 1.0;
                    f = mx;
                    if (act[m] && t == 0) {
                        op.scaleWrite[p] = logScalers ? log(mx) : mx;
                    }
                } else {
                    f = act[m] ? op.scaleRead[p] : 1.0;
                    if (logScalers) f = exp(f);
                }
                if (act[m]) {
                    const double inv = 1.0 / f;
                    for (int cc = 0; cc < C; ++cc) {
                        double* drow = op.dest + ((size_t)cc * Ppad + p) * Sp + 2 * t;
#pragma unroll
                        for (int n = 0; n < NT; ++n) {
                            double2 v = *reinterpret_cast<double2*>(drow + 8 * n);
                            v.x *= inv; v.y *= inv;
                            *reinterpret_cast<double2*>(drow + 8 * n) = v;
                        }
                    }
                }
            }
        }
        // (a) every warp is done with this buffer before the copy issued next iteration overwrites it,
        // (b) rows written by other lanes of this warp become visible to the next op's A-fragment loads
        if (cg == cb - 1 || c == C - 1) __syncthreads();
    }
}

template <int NT, int WARPS, bool PRE = false, int MT = 2>
static cudaError_t launchWalkMmaT(Instance* in, const DevOp* dOps, const int4* dSubs, int nSubs, int maxWindow) {
    constexpr int Sp = 8 * NT;
    constexpr int TILE = WARPS * 8 * MT;             // patterns per block
    const size_t pair = 2 * (size_t)Sp * (Sp + 4) * sizeof(double);
    // as many categories per staging round as keep three blocks resident per SM (72 KB each)
    const int cb = (int)std::max<size_t>(1, std::min<size_t>((size_t)in->C, (72 * 1024) / pair));
    const size_t smem = pair * cb;
    dim3 grid((maxWindow + TILE - 1) / TILE, nSubs);
    if constexpr (MT == 2) {
        // a thin phase (the walks near the root: fewer blocks than two per SM) runs with 8-pattern warp tiles: twice the blocks
        if (!PRE && (long)grid.x * nSubs < 2L * in->smCount && in->thinR1)
            return launchWalkMmaT<NT, WARPS, PRE, PRE ? 2 : 1>(in, dOps, dSubs, nSubs, maxWindow);
    }
    const int slot = (PRE ? 1 : 0) + (MT == 1 ? 4 : 0);
    if (cb == 1) {
        if (smem > in->mmaSmemConfigured[slot]) {
            cudaError_t e = cudaFuncSetAttribute(k_walk_mma<NT, WARPS, PRE, false, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
            in->mmaSmemConfigured[slot] = smem;
        }
        k_walk_mma<NT, WARPS, PRE, false, MT><<<grid, WARPS * 32, smem, in->stream>>>(dOps, dSubs, in->S, in->C, in->Ppad, in->logScalers ? 1 : 0, 1);
    } else {
        if (smem > in->mmaSmemConfigured[slot + 2]) {
            cudaError_t e = cudaFuncSetAttribute(k_walk_mma<NT, WARPS, PRE, true, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
            in->mmaSmemConfigured[slot + 2] = smem;
        }
        k_walk_mma<NT, WARPS, PRE, true, MT><<<grid, WARPS * 32, smem, in->stream>>>(dOps, dSubs, in->S, in->C, in->Ppad, in->logScalers ? 1 : 0, cb);
    }
    return cudaGetLastError();
}

cudaError_t launchWalkGeneric(Instance* in, const DevOp* dOps, const int4* dSubs, int nSubs, int maxWindow, bool preOrder) {
    if (nSubs <= 0) return cudaSuccess;
    if (in->genericMma && preOrder) {
        switch (in->Sp / 8) {
            case 1: return launchWalkMmaT<1, 4, true>(in, dOps, dSubs, nSubs, maxWindow);
            case 2: return launchWalkMmaT<2, 4, true>(in, dOps, dSubs, nSubs, maxWindow);
            case 3: return launchWalkMmaT<3, 4, true>(in, dOps, dSubs, nSubs, maxWindow);
            case 4: return launchWalkMmaT<4, 4, true>(in, dOps, dSubs, nSubs, maxWindow);
            case 8: return launchWalkMmaT<8, 4, true>(in, dOps, dSubs, nSubs, maxWindow);
            default: break;
        }
    } else if (in->genericMma) {
        switch (in->Sp / 8) {
            case 1: return launchWalkMmaT<1, 4>(in, dOps, dSubs, nSubs, maxWindow);
            case 2: return launchWalkMmaT<2, 4>(in, dOps, dSubs, nSubs, maxWindow);
            case 3: return launchWalkMmaT<3, 4>(in, dOps, dSubs, nSubs, maxWindow);
            case 4: return launchWalkMmaT<4, 4>(in, dOps, dSubs, nSubs, maxWindow);
            case 8: return launchWalkMmaT<8, 4>(in, dOps, dSubs, nSubs, maxWindow);
            default: break;      // other state counts: FMA block walk below
        }
    }
    const int Sp = in->Sp;
    const size_t budget = in->maxSmemOptin > 16384 ? in->maxSmemOptin - 2048 : 46000;
    const int tiles = preOrder ? 3 : 2;
    int stage = (2 * (size_t)Sp * Sp * 8 + (size_t)tiles * 8 * (size_t)Sp * 8 + 64 <= budget) ? 1 : 0;
    size_t fixed = stage ? 2 * (size_t)Sp * Sp * 8 : 0;
    int TP = 32;
    while (TP > 1 && fixed + (size_t)TP * (tiles * Sp + 1) * 8 > budget) TP >>= 1;
    while (TP > 8 && (in->Ppad + TP - 1) / TP < in->smCount) TP >>= 1;   // keep every SM busy
    size_t smem = fixed + (size_t)TP * (tiles * Sp + 1) * 8;
    if (smem > in->genericSmemConfigured) {
        cudaError_t e = cudaFuncSetAttribute(k_walk_generic, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        in->genericSmemConfigured = smem;
    }
    dim3 grid((maxWindow + TP - 1) / TP, nSubs);
    k_walk_generic<<<grid, 256, smem, in->stream>>>(dOps, dSubs, in->S, Sp, in->C, in->Ppad, TP,
                                                      in->logScalers ? 1 : 0, stage, preOrder ? 1 : 0);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// edge derivatives (pre-order route): one block per edge, thread per pattern
// ---------------------------------------------------------------------------------------------
// d[e,p] = (sum_c w_c sum_j pre[c,p,j] (D_c post)[c,p,j]) / (sum_c w_c sum_j pre[c,p,j] post[c,p,j])
// (preorder/AbstractBeagleBranchGradientDelegate.java:97-150 states the same reduction in Java).
// T = the partials' storage type (float on a PRECISION_SINGLE instance with S < 4)
template <typename T>
__device__ __forceinline__ void edgeDerivativesBody(const EdgeRefT<T>* __restrict__ edges, const double* __restrict__ weights,
                                                    const double* __restrict__ patternWeights, int S, int Sp, int C, int P,
                                                    int Ppad, int matCP, int stageD, double* __restrict__ outPerPattern,
                                                    double* __restrict__ outSum, double* __restrict__ outSumSq) {
    extern __shared__ double smd[];            // D_c[j][k] row-major for all categories (when it fits)
    __shared__ double red1[256], red2[256];
    const EdgeRefT<T> e = edges[blockIdx.x];
    const int tid = threadIdx.x;
    auto dIndex = [&](int c, int j, int k) -> size_t {       // location of D[c][j][k] in the engine's matrix layouts
        return matCP ? ((size_t)k * matCP + c) * 4 + j : ((size_t)c * Sp + k) * Sp + j;
    };
    if (stageD) {
        for (int q = tid; q < C * S * S; q += 256) {
            const int c = q / (S * S), r = q % (S * S);
            smd[q] = e.D[dIndex(c, r / S, r % S)];
        }
        __syncthreads();
    }
    double acc1 = 0.0, acc2 = 0.0;
    for (int p = tid; p < P; p += 256) {
        double num = 0.0, den = 0.0;
        const int s = e.states ? e.states[p] : -1;
        for (int c = 0; c < C; ++c) {
            const T* pre = e.pre + ((size_t)c * Ppad + p) * Sp;
            const T* post = e.post ? e.post + ((size_t)c * Ppad + p) * Sp : nullptr;
            double nc = 0.0, dc = 0.0;
            for (int j = 0; j < S; ++j) {
                double dp = 0.0, pj;
                if (post) {
                    for (int k2 = 0; k2 < S; ++k2)
                        dp += (stageD ? smd[((size_t)c * S + j) * S + k2] : e.D[dIndex(c, j, k2)]) * post[k2];
                    pj = post[j];
                } else if (s < S) {
                    dp = stageD ? smd[((size_t)c * S + j) * S + s] : e.D[dIndex(c, j, s)];
                    pj = (j == s) ? 1.0 : 0.0;
                } else {
                    for (int k2 = 0; k2 < S; ++k2) dp += stageD ? smd[((size_t)c * S + j) * S + k2] : e.D[dIndex(c, j, k2)];
                    pj = 1.0;
                }
                nc += pre[j] * dp;
                dc += pre[j] * pj;
            }
            num += weights[c] * nc;
            den += weights[c] * dc;
        }
        const double d = num / den;
        if (outPerPattern) outPerPattern[(size_t)blockIdx.x * P + p] = d;
        acc1 += patternWeights[p] * d;
        acc2 += patternWeights[p] * d * d;
    }
    red1[tid] = acc1; red2[tid] = acc2;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (tid < w) { red1[tid] += red1[tid + w]; red2[tid] += red2[tid + w]; }
        __syncthreads();
    }
    if (tid == 0) { outSum[blockIdx.x] = red1[0]; outSumSq[blockIdx.x] = red2[0]; }
}

__global__ void __launch_bounds__(256)
k_edge_derivatives(const EdgeRef* __restrict__ edges, const double* __restrict__ weights,
                   const double* __restrict__ patternWeights, int S, int Sp, int C, int P, int Ppad, int matCP,
                   int stageD, double* __restrict__ outPerPattern, double* __restrict__ outSum,
                   double* __restrict__ outSumSq) {
    edgeDerivativesBody<double>(edges, weights, patternWeights, S, Sp, C, P, Ppad, matCP, stageD, outPerPattern, outSum,
                                outSumSq);
}

__global__ void __launch_bounds__(256)
k_edge_derivatives_f32(const EdgeRefT<float>* __restrict__ edges, const double* __restrict__ weights,
                       const double* __restrict__ patternWeights, int S, int Sp, int C, int P, int Ppad, int matCP,
                       int stageD, double* __restrict__ outPerPattern, double* __restrict__ outSum,
                       double* __restrict__ outSumSq) {
    edgeDerivativesBody<float>(edges, weights, patternWeights, S, Sp, C, P, Ppad, matCP, stageD, outPerPattern, outSum,
                               outSumSq);
}

// 4-state form: grid (256-pattern chunks, edges), a thread owns one (edge, pattern); the C differential matrices of the
// edge sit in shared memory, the 2 C cell loads of a thread are issued four categories at a time.
template <typename T>
__device__ __forceinline__ void edgeDerivatives4Body(const EdgeRefT<T>* __restrict__ edges, const double* __restrict__ weights,
                                                     const double* __restrict__ patternWeights, int C, int P, int Ppad,
                                                     int matCP, double* __restrict__ outPerPattern,
                                                     double* __restrict__ partial) {
    extern __shared__ double sD[];                  // [C][j][k]
    __shared__ double red[8][2];
    const EdgeRefT<T> e = edges[blockIdx.y];
    const int tid = threadIdx.x, p = blockIdx.x * 256 + tid;
    for (int q = tid; q < C * 16; q += 256) {
        const int c = q >> 4, j = (q >> 2) & 3, k = q & 3;
        sD[q] = e.D[((size_t)k * matCP + c) * 4 + j];
    }
    __syncthreads();
    double s1 = 0.0, s2 = 0.0;
    if (p < P) {
        const int s = e.states ? e.states[p] : -1;
        double num = 0.0, den = 0.0;
        for (int c0 = 0; c0 < C; c0 += 4) {
            double a[4][4], b[4][4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const size_t off = ((size_t)min(c0 + u, C - 1) * Ppad + p) * 4;
                loadCellRo(e.pre + off, a[u]);
                if (e.post) loadCellRo(e.post + off, b[u]);
                else {
#pragma unroll
                    for (int j = 0; j < 4; ++j) b[u][j] = (s >= 4 || s == j) ? 1.0 : 0.0;
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (c0 + u >= C) break;
                const double* D = sD + (c0 + u) * 16;
                double nc = 0.0, dc = 0.0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const double v = D[j * 4] * b[u][0] + D[j * 4 + 1] * b[u][1] + D[j * 4 + 2] * b[u][2] + D[j * 4 + 3] * b[u][3];
                    nc += a[u][j] * v;
                    dc += a[u][j] * b[u][j];
                }
                num += weights[c0 + u] * nc;
                den += weights[c0 + u] * dc;
            }
        }
        const double d = num / den;
        if (outPerPattern) outPerPattern[(size_t)blockIdx.y * P + p] = d;
        s1 = patternWeights[p] * d;
        s2 = patternWeights[p] * d * d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if ((tid & 31) == 0) { red[tid >> 5][0] = s1; red[tid >> 5][1] = s2; }
    __syncthreads();
    if (tid < 2) {
        double r = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) r += red[w][tid];
        partial[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 2 + tid] = r;
    }
}

__global__ void __launch_bounds__(256)
k_edge_derivatives4(const EdgeRef* __restrict__ edges, const double* __restrict__ weights,
                    const double* __restrict__ patternWeights, int C, int P, int Ppad, int matCP,
                    double* __restrict__ outPerPattern, double* __restrict__ partial) {
    edgeDerivatives4Body<double>(edges, weights, patternWeights, C, P, Ppad, matCP, outPerPattern, partial);
}

__global__ void __launch_bounds__(256)
k_edge_derivatives4_f32(const EdgeRefT<float>* __restrict__ edges, const double* __restrict__ weights,
                        const double* __restrict__ patternWeights, int C, int P, int Ppad, int matCP,
                        double* __restrict__ outPerPattern, double* __restrict__ partial) {
    edgeDerivatives4Body<float>(edges, weights, patternWeights, C, P, Ppad, matCP, outPerPattern, partial);
}

// Tensor-pipe form for the state counts of the DMMA walk (Sp = 8 NT): block = 4 warps x 16 patterns of ONE edge.
// Per category the row-major D_c is staged like a transition matrix, v = D_c post is the same m8n8k4 contraction as a
// post-order child term, and the two dot products with the pre-order partial are taken in the accumulator layout.
// Block partial sums go to `partial[(edge * tiles + tile) * 2 + {0,1}]`; k_edge_sum adds them in tile order.
template <int NT>
__global__ void __launch_bounds__(128)
k_edge_derivatives_mma(const EdgeRef* __restrict__ edges, const double* __restrict__ weights,
                       const double* __restrict__ patternWeights, int S, int C, int P, int Ppad,
                       double* __restrict__ outPerPattern, double* __restrict__ partial) {
    constexpr int Sp = 8 * NT;
    constexpr int LD = Sp + 4;
    extern __shared__ double smm[];                  // [Sp][LD]
    __shared__ double red[4][2];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const EdgeRef e = edges[blockIdx.y];
    const int pw = blockIdx.x * 64 + w * 16;
    const size_t mRow = (size_t)C * Sp * Sp;
    bool act[2];
    int st[2] = {0, 0};
    double num[2] = {0.0, 0.0}, den[2] = {0.0, 0.0};
#pragma unroll
    for (int m = 0; m < 2; ++m) {
        act[m] = pw + 8 * m + g < P;
        if (e.states != nullptr && act[m]) st[m] = e.states[pw + 8 * m + g];
    }
    for (int c = 0; c < C; ++c) {
        __syncthreads();                             // everyone is done with the previous category's matrix
        const double* gD = e.D + mRow + (size_t)c * Sp * LD;      // padded row-major copy: already in the shared-memory shape
        for (int q = tid; q < Sp * LD / 2; q += 128) cpAsync16(smm + 2 * q, gD + 2 * q);
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        double v[2][NT][2];
        if (e.post != nullptr) {
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int n = 0; n < NT; ++n) { v[m][n][0] = 0.0; v[m][n][1] = 0.0; }
            // branch-free A operands ahead of the .aligned mma.sync: see the pre-order form of k_walk_mma
            const double* xrow0 = e.post + ((size_t)c * Ppad + min(pw + g, Ppad - 1)) * Sp + t;
            const double* xrow1 = e.post + ((size_t)c * Ppad + min(pw + 8 + g, Ppad - 1)) * Sp + t;
            const double* brow = smm + g * LD + t;
#pragma unroll 4
            for (int kc = 0; kc < Sp / 4; ++kc) {
                const double x0 = xrow0[4 * kc], x1 = xrow1[4 * kc];
                const double a0 = selOn(x0, act[0]), a1 = selOn(x1, act[1]);
#pragma unroll
                for (int n = 0; n < NT; ++n) {
                    const double b = brow[n * 8 * LD + 4 * kc];
                    dmma884acc(v[0][n][0], v[0][n][1], a0, b);
                    dmma884acc(v[1][n][0], v[1][n][1], a1, b);
                }
            }
        } else {
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int n = 0; n < NT; ++n)
#pragma unroll
                    for (int x = 0; x < 2; ++x) {
                        const int i = 8 * n + 2 * t + x;
                        double d = 0.0;
                        if (st[m] < S) d = smm[i * LD + st[m]];
                        else for (int k = 0; k < S; ++k) d += smm[i * LD + k];
                        v[m][n][x] = d;
                    }
        }
        const double wc = weights[c];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
            if (!act[m]) continue;
            const size_t off = ((size_t)c * Ppad + (pw + 8 * m + g)) * Sp + 2 * t;
            double nn = 0.0, dd = 0.0;
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                const double2 a = *reinterpret_cast<const double2*>(e.pre + off + 8 * n);
                nn += a.x * v[m][n][0] + a.y * v[m][n][1];
                if (e.post != nullptr) {
                    const double2 b = *reinterpret_cast<const double2*>(e.post + off + 8 * n);
                    dd += a.x * b.x + a.y * b.y;
                } else {
                    const int i = 8 * n + 2 * t;
                    if (st[m] >= S) dd += (i < S ? a.x : 0.0) + (i + 1 < S ? a.y : 0.0);
                    else dd += (i == st[m] ? a.x : 0.0) + (i + 1 == st[m] ? a.y : 0.0);
                }
            }
            num[m] += wc * nn;
            den[m] += wc * dd;
        }
    }
    double s1 = 0.0, s2 = 0.0;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
        double nn = num[m], dd = den[m];
        nn += __shfl_xor_sync(0xffffffffu, nn, 1); nn += __shfl_xor_sync(0xffffffffu, nn, 2);
        dd += __shfl_xor_sync(0xffffffffu, dd, 1); dd += __shfl_xor_sync(0xffffffffu, dd, 2);
        if (act[m] && t == 0) {
            const int p = pw + 8 * m + g;
            const double d = nn / dd;
            if (outPerPattern) outPerPattern[(size_t)blockIdx.y * P + p] = d;
            s1 += patternWeights[p] * d;
            s2 += patternWeights[p] * d * d;
        }
    }
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) { red[w][0] = s1; red[w][1] = s2; }
    __syncthreads();
    if (tid < 2) {
        const double r = red[0][tid] + red[1][tid] + red[2][tid] + red[3][tid];
        partial[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 2 + tid] = r;
    }
}

__global__ void __launch_bounds__(128)
k_edge_sum(const double* __restrict__ partial, int tiles, int count, double* __restrict__ outSum,
           double* __restrict__ outSumSq) {
    const int e = blockIdx.x * 128 + threadIdx.x;
    if (e >= count) return;
    double s1 = 0.0, s2 = 0.0;
    for (int k = 0; k < tiles; ++k) { s1 += partial[((size_t)e * tiles + k) * 2]; s2 += partial[((size_t)e * tiles + k) * 2 + 1]; }
    outSum[e] = s1;
    outSumSq[e] = s2;
}

template <int NT>
static cudaError_t launchEdgeMmaT(Instance* in, const EdgeRef* dEdges, int count, const double* weights,
                                  double* outPerPattern, double* outSum, double* outSumSq, double* partial) {
    constexpr int Sp = 8 * NT;
    const size_t smem = (size_t)Sp * (Sp + 4) * sizeof(double);
    const int tiles = (in->P + 63) / 64;
    dim3 grid(tiles, count);
    k_edge_derivatives_mma<NT><<<grid, 128, smem, in->stream>>>(dEdges, weights, in->dPatternWeights, in->S, in->C,
                                                                in->P, in->Ppad, outPerPattern, partial);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    k_edge_sum<<<(count + 127) / 128, 128, 0, in->stream>>>(partial, tiles, count, outSum, outSumSq);
    return cudaGetLastError();
}

// doubles of workspace the tensor-pipe form needs (0 = this state count uses the plain kernel)
size_t edgeDerivativeWorkspace(const Instance* in, int count) {
    if (count > 65535) return 0;
    if (in->matCP > 0 && in->S == 4) return (size_t)count * ((in->P + 255) / 256) * 2;
    const int nt = in->Sp / 8;
    const bool mma = in->genericMma && in->matCP == 0 && in->Sp % 8 == 0 && ((nt >= 1 && nt <= 4) || nt == 8);
    return mma ? (size_t)count * ((in->P + 63) / 64) * 2 : 0;
}

cudaError_t launchEdgeDerivatives(Instance* in, const EdgeRefT<void>* dRefs, int count, const double* weights,
                                  double* outPerPattern, double* outSum, double* outSumSq, double* partial) {
    const EdgeRef* dEdges = reinterpret_cast<const EdgeRef*>(dRefs);
    const EdgeRefT<float>* dEdgesF = reinterpret_cast<const EdgeRefT<float>*>(dRefs);
    if (partial != nullptr && in->matCP > 0) {
        const int chunks = (in->P + 255) / 256;
        const dim3 grid(chunks, count);
        if (in->single)
            k_edge_derivatives4_f32<<<grid, 256, sizeof(double) * 16 * in->C, in->stream>>>(
                dEdgesF, weights, in->dPatternWeights, in->C, in->P, in->Ppad, in->matCP, outPerPattern, partial);
        else
            k_edge_derivatives4<<<grid, 256, sizeof(double) * 16 * in->C, in->stream>>>(
                dEdges, weights, in->dPatternWeights, in->C, in->P, in->Ppad, in->matCP, outPerPattern, partial);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        k_edge_sum<<<(count + 127) / 128, 128, 0, in->stream>>>(partial, chunks, count, outSum, outSumSq);
        return cudaGetLastError();
    }
    if (partial != nullptr) {
        switch (in->Sp / 8) {
            case 1: return launchEdgeMmaT<1>(in, dEdges, count, weights, outPerPattern, outSum, outSumSq, partial);
            case 2: return launchEdgeMmaT<2>(in, dEdges, count, weights, outPerPattern, outSum, outSumSq, partial);
            case 3: return launchEdgeMmaT<3>(in, dEdges, count, weights, outPerPattern, outSum, outSumSq, partial);
            case 4: return launchEdgeMmaT<4>(in, dEdges, count, weights, outPerPattern, outSum, outSumSq, partial);
            case 8: return launchEdgeMmaT<8>(in, dEdges, count, weights, outPerPattern, outSum, outSumSq, partial);
            default: break;
        }
    }
    const size_t need = (size_t)in->C * in->S * in->S * sizeof(double);
    const size_t budget = in->maxSmemOptin > 16384 ? in->maxSmemOptin - 8192 : 40000;
    const int stageD = need <= budget ? 1 : 0;
    const size_t smem = stageD ? need : 0;
    if (in->single) {                  // S < 4 (S = 4 took the form above); C <= 8 keeps smem small
        k_edge_derivatives_f32<<<count, 256, smem, in->stream>>>(dEdgesF, weights, in->dPatternWeights, in->S, in->Sp, in->C,
                                                                 in->P, in->Ppad, in->matCP, stageD, outPerPattern, outSum,
                                                                 outSumSq);
        return cudaGetLastError();
    }
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(k_edge_derivatives, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    k_edge_derivatives<<<count, 256, smem, in->stream>>>(dEdges, weights, in->dPatternWeights, in->S, in->Sp, in->C,
                                                         in->P, in->Ppad, in->matCP, stageD, outPerPattern, outSum, outSumSq);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// cross-product differentials (SubstitutionModelCrossProductDelegate.java:140-181 is the caller):
//   out[i][j] += sum_edges t_e sum_p w_p ( sum_c weight_c rate_c pre_c[p][i] post_c[p][j] ) / ( sum_c weight_c pre_c[p].post_c[p] )
// both partials sit at the child end of the branch, so sum_ij out[i][j] Q[i][j] = d logL / d(log of a common factor on
// every branch length) exactly (the identity AbstractLogAdditiveSubstitutionModelGradient.java:220-227 relies on).
// Two-stage and deterministic: every block leaves its S x S partial in `scratch`, k_cross_reduce adds them in a
// fixed order.
// ---------------------------------------------------------------------------------------------
// 4-state: a thread owns a pattern, the 16 accumulators stay in registers across the block's edges.
template <typename T>
__device__ __forceinline__ void cross4Body(const EdgeRefT<T>* __restrict__ edges, int count, const double* __restrict__ rates,
                                           const double* __restrict__ weights, const double* __restrict__ patternWeights,
                                           int C, int P, int Ppad, double* __restrict__ scratch) {
    __shared__ double red[8][16];
    const int tid = threadIdx.x, p = blockIdx.x * 256 + tid;
    double acc[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) acc[q] = 0.0;
    if (p < P) {
        const double wp = patternWeights[p];
        for (int e = blockIdx.y; e < count; e += gridDim.y) {
            const EdgeRefT<T> r = edges[e];
            const int s = r.states ? r.states[p] : -1;
            double num[16], den = 0.0;
#pragma unroll
            for (int q = 0; q < 16; ++q) num[q] = 0.0;
            // four categories per round, clamped + zero-weighted past C: all 8 loads of a round are in flight together
            for (int c0 = 0; c0 < C; c0 += 4) {
                double a[4][4], b[4][4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const size_t off = ((size_t)min(c0 + u, C - 1) * Ppad + p) * 4;
                    loadCellRo(r.pre + off, a[u]);
                    if (r.post) loadCellRo(r.post + off, b[u]);
                    else {
#pragma unroll
                        for (int j = 0; j < 4; ++j) b[u][j] = (s >= 4 || s == j) ? 1.0 : 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const bool live = c0 + u < C;
                    const double wc = live ? weights[c0 + u] : 0.0, f = live ? wc * rates[c0 + u] : 0.0;
                    den += wc * (a[u][0] * b[u][0] + a[u][1] * b[u][1] + a[u][2] * b[u][2] + a[u][3] * b[u][3]);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const double fa = f * a[u][i];
#pragma unroll
                        for (int j = 0; j < 4; ++j) num[i * 4 + j] += fa * b[u][j];
                    }
                }
            }
            const double sc = wp * r.len / den;
#pragma unroll
            for (int q = 0; q < 16; ++q) acc[q] += sc * num[q];
        }
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        double v = acc[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((tid & 31) == 0) red[tid >> 5][q] = v;
    }
    __syncthreads();
    if (tid < 16) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) v += red[w][tid];
        scratch[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 16 + tid] = v;
    }
}

__global__ void __launch_bounds__(256)
k_cross4(const EdgeRef* __restrict__ edges, int count, const double* __restrict__ rates,
         const double* __restrict__ weights, const double* __restrict__ patternWeights, int C, int P, int Ppad,
         double* __restrict__ scratch) {
    cross4Body<double>(edges, count, rates, weights, patternWeights, C, P, Ppad, scratch);
}

__global__ void __launch_bounds__(256)
k_cross4_f32(const EdgeRefT<float>* __restrict__ edges, int count, const double* __restrict__ rates,
             const double* __restrict__ weights, const double* __restrict__ patternWeights, int C, int P, int Ppad,
             double* __restrict__ scratch) {
    cross4Body<float>(edges, count, rates, weights, patternWeights, C, P, Ppad, scratch);
}

// any state count: a block owns PCH patterns; per (edge, category) the scaled pre tile and the post tile go through
// shared memory and every thread keeps a 4 x 4 tile of the S x S outer-product sum in registers.
// (also the 4-state form for S < 4, k_cross4 being S = 4 only; T = float on a PRECISION_SINGLE instance)
template <typename T>
__device__ __forceinline__ void crossGenericBody(const EdgeRefT<T>* __restrict__ edges, int count,
                                                 const double* __restrict__ rates, const double* __restrict__ weights,
                                                 const double* __restrict__ patternWeights, int S, int Sp, int C, int P,
                                                 int Ppad, int PCH, double* __restrict__ scratch) {
    extern __shared__ double smx[];
    const int S4 = (S + 3) & ~3, nt = S4 / 4, ntiles = nt * nt;
    double* fp = smx;                       // [PCH]  w_p t_e / den_p
    double* spre = smx + ((PCH + 1) & ~1);  // [PCH][S4], 16-byte aligned for the double2 reads
    double* spost = spre + (size_t)PCH * S4;
    const int tid = threadIdx.x, p0 = blockIdx.x * PCH, np = min(PCH, P - p0);
    double* mine = scratch + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * S * S;
    for (int tb = 0; tb < ntiles; tb += 256) {
        const int tile = tb + tid;
        const bool active = tile < ntiles;
        const int ti = active ? tile / nt : 0, tj = active ? tile % nt : 0;
        double acc[4][4];
#pragma unroll
        for (int x = 0; x < 4; ++x)
#pragma unroll
            for (int y = 0; y < 4; ++y) acc[x][y] = 0.0;
        for (int e = blockIdx.y; e < count; e += gridDim.y) {
            const EdgeRefT<T> r = edges[e];
            {   // den_p: 8 lanes per pattern, fixed-order shuffle reduction
                const int pp = tid >> 3, lane = tid & 7;
                for (int base = 0; base < np; base += 32) {
                    const int q = base + pp;
                    double d = 0.0;
                    if (q < np) {
                        const int p = p0 + q;
                        const int s = r.states ? r.states[p] : -1;
                        for (int c = 0; c < C; ++c) {
                            const T* pre = r.pre + ((size_t)c * Ppad + p) * Sp;
                            double dc = 0.0;
                            if (r.post) {
                                const T* post = r.post + ((size_t)c * Ppad + p) * Sp;
                                for (int k = lane; k < S; k += 8) dc += pre[k] * post[k];
                            } else if (s < S) {
                                if (lane == (s & 7)) dc = pre[s];
                            } else {
                                for (int k = lane; k < S; k += 8) dc += pre[k];
                            }
                            d += weights[c] * dc;
                        }
                    }
                    d += __shfl_xor_sync(0xffffffffu, d, 4);
                    d += __shfl_xor_sync(0xffffffffu, d, 2);
                    d += __shfl_xor_sync(0xffffffffu, d, 1);
                    if (q < np && lane == 0) fp[q] = patternWeights[p0 + q] * r.len / d;
                }
            }
            __syncthreads();
            for (int c = 0; c < C; ++c) {
                const double f = weights[c] * rates[c];
                for (int idx = tid; idx < np * S4; idx += 256) {
                    const int pp = idx / S4, k = idx - pp * S4, p = p0 + pp;
                    double a = 0.0, b = 0.0;
                    if (k < S) {
                        a = r.pre[((size_t)c * Ppad + p) * Sp + k] * fp[pp] * f;
                        if (r.post) b = r.post[((size_t)c * Ppad + p) * Sp + k];
                        else { const int s = r.states[p]; b = (s >= S || s == k) ? 1.0 : 0.0; }
                    }
                    spre[idx] = a;
                    spost[idx] = b;
                }
                __syncthreads();
                if (active) {
                    for (int pp = 0; pp < np; ++pp) {
                        const double2* pa = reinterpret_cast<const double2*>(spre + (size_t)pp * S4 + ti * 4);
                        const double2* pb = reinterpret_cast<const double2*>(spost + (size_t)pp * S4 + tj * 4);
                        const double2 a0 = pa[0], a1 = pa[1], b0 = pb[0], b1 = pb[1];
                        const double a[4] = {a0.x, a0.y, a1.x, a1.y}, b[4] = {b0.x, b0.y, b1.x, b1.y};
#pragma unroll
                        for (int x = 0; x < 4; ++x)
#pragma unroll
                            for (int y = 0; y < 4; ++y) acc[x][y] += a[x] * b[y];
                    }
                }
                __syncthreads();
            }
        }
        if (active) {
#pragma unroll
            for (int x = 0; x < 4; ++x)
#pragma unroll
                for (int y = 0; y < 4; ++y) {
                    const int i = ti * 4 + x, j = tj * 4 + y;
                    if (i < S && j < S) mine[(size_t)i * S + j] = acc[x][y];
                }
        }
    }
}

__global__ void __launch_bounds__(256)
k_cross_generic(const EdgeRef* __restrict__ edges, int count, const double* __restrict__ rates,
                const double* __restrict__ weights, const double* __restrict__ patternWeights, int S, int Sp, int C,
                int P, int Ppad, int PCH, double* __restrict__ scratch) {
    crossGenericBody(edges, count, rates, weights, patternWeights, S, Sp, C, P, Ppad, PCH, scratch);
}

__global__ void __launch_bounds__(256)
k_cross_generic_f32(const EdgeRefT<float>* __restrict__ edges, int count, const double* __restrict__ rates,
                    const double* __restrict__ weights, const double* __restrict__ patternWeights, int S, int Sp, int C,
                    int P, int Ppad, int PCH, double* __restrict__ scratch) {
    crossGenericBody(edges, count, rates, weights, patternWeights, S, Sp, C, P, Ppad, PCH, scratch);
}

// Tensor-pipe form for Sp = 8 NT: out[i][j] += sum_p A[p][i] B[p][j] is a GEMM whose contraction index is the pattern.
// Block = one 32-pattern tile x a group of edges, 4 warps; per (edge, category) the scaled pre tile (A) and the post tile
// (B) are staged in shared memory with the (Sp+4) row stride, warp w owns output rows 8(w + 4 mi) .. +7 and all columns:
// lane (g,t) feeds A[i = 8m+g][k = t] and B[k = t][j = 8n+g] of every 4-pattern chunk to one m8n8k4 DMMA.
template <int NT>
__global__ void __launch_bounds__(128, 4)
k_cross_mma(const EdgeRef* __restrict__ edges, int count, const double* __restrict__ rates,
            const double* __restrict__ weights, const double* __restrict__ patternWeights, int S, int C, int P,
            int Ppad, double* __restrict__ scratch) {
    constexpr int Sp = 8 * NT, LDs = Sp + 4, TP = 32, MT = (NT + 3) / 4;
    extern __shared__ double smc[];
    double* sA = smc;                        // [TP][LDs]  w_p t_e / den_p * w_c r_c * pre
    double* sB = smc + TP * LDs;             // [TP][LDs]  post
    double* fp = sB + TP * LDs;              // [TP]
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, g = lane >> 2, t = lane & 3;
    const int p0 = blockIdx.x * TP, np = min(TP, P - p0);
    double acc[MT][NT][2];
#pragma unroll
    for (int mi = 0; mi < MT; ++mi)
#pragma unroll
        for (int n = 0; n < NT; ++n) { acc[mi][n][0] = 0.0; acc[mi][n][1] = 0.0; }
    for (int e = blockIdx.y; e < count; e += gridDim.y) {
        const EdgeRef r = edges[e];
        {   // per-pattern factor: 8 lanes per pattern, fixed-order shuffle reduction (fp is free: the last MMA pass synced).
            // Fully unrolled with predicated loads: all 2 NT loads of a lane are in flight together (a rolled loop
            // serialised one L2 round trip per 8 states and made this pass the whole kernel's critical path).
            const int pp = tid >> 3, l8 = tid & 7;
#pragma unroll
            for (int base = 0; base < TP; base += 16) {
                const int q = base + pp;
                double d = 0.0;
                if (q < np) {
                    const int p = p0 + q;
                    const int s = r.states ? r.states[p] : -1;
                    for (int c = 0; c < C; ++c) {
                        const double* pre = r.pre + ((size_t)c * Ppad + p) * Sp;
                        const double* post = r.post ? r.post + ((size_t)c * Ppad + p) * Sp : nullptr;
                        double x[NT], y[NT];
#pragma unroll
                        for (int u = 0; u < NT; ++u) {
                            const int k = l8 + 8 * u;
                            x[u] = k < S ? pre[k] : 0.0;
                            y[u] = post ? post[k] : ((s >= S || s == k) ? 1.0 : 0.0);
                        }
                        double dc = 0.0;
#pragma unroll
                        for (int u = 0; u < NT; ++u) dc += x[u] * y[u];
                        d += weights[c] * dc;
                    }
                }
                d += __shfl_xor_sync(0xffffffffu, d, 4);
                d += __shfl_xor_sync(0xffffffffu, d, 2);
                d += __shfl_xor_sync(0xffffffffu, d, 1);
                if (l8 == 0) fp[q] = q < np ? patternWeights[p0 + q] * r.len / d : 0.0;
            }
        }
        __syncthreads();
        for (int c = 0; c < C; ++c) {
            const double f = weights[c] * rates[c];
            for (int q2 = tid; q2 < TP * Sp / 2; q2 += 128) {
                const int pp = (2 * q2) / Sp, k = (2 * q2) % Sp;
                double2 a = make_double2(0.0, 0.0), b = make_double2(0.0, 0.0);
                if (pp < np) {
                    const size_t off = ((size_t)c * Ppad + p0 + pp) * Sp + k;
                    const double sc = fp[pp] * f;
                    a = *reinterpret_cast<const double2*>(r.pre + off);
                    a.x = k < S ? a.x * sc : 0.0;
                    a.y = k + 1 < S ? a.y * sc : 0.0;
                    if (r.post) {
                        b = *reinterpret_cast<const double2*>(r.post + off);
                        if (k >= S) b.x = 0.0;
                        if (k + 1 >= S) b.y = 0.0;
                    } else {
                        const int s = r.states[p0 + pp];
                        b.x = (k < S && (s >= S || s == k)) ? 1.0 : 0.0;
                        b.y = (k + 1 < S && (s >= S || s == k + 1)) ? 1.0 : 0.0;
                    }
                }
                *reinterpret_cast<double2*>(sA + pp * LDs + k) = a;
                *reinterpret_cast<double2*>(sB + pp * LDs + k) = b;
            }
            __syncthreads();
#pragma unroll 2
            for (int kc = 0; kc < TP / 4; ++kc) {
                const double* arow = sA + (4 * kc + t) * LDs + g;
                const double* brow = sB + (4 * kc + t) * LDs + g;
                double a[MT];
#pragma unroll
                for (int mi = 0; mi < MT; ++mi) a[mi] = (w + 4 * mi < NT) ? arow[8 * (w + 4 * mi)] : 0.0;
#pragma unroll
                for (int n = 0; n < NT; ++n) {
                    const double b = brow[8 * n];
#pragma unroll
                    for (int mi = 0; mi < MT; ++mi)
                        if (w + 4 * mi < NT) dmma884acc(acc[mi][n][0], acc[mi][n][1], a[mi], b);
                }
            }
            __syncthreads();
        }
    }
    double* mine = scratch + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * S * S;
#pragma unroll
    for (int mi = 0; mi < MT; ++mi) {
        const int m = w + 4 * mi, i = 8 * m + g;
        if (m >= NT || i >= S) continue;
#pragma unroll
        for (int n = 0; n < NT; ++n) {
            const int j = 8 * n + 2 * t;
            if (j < S) mine[(size_t)i * S + j] = acc[mi][n][0];
            if (j + 1 < S) mine[(size_t)i * S + j + 1] = acc[mi][n][1];
        }
    }
}

template <int NT>
static cudaError_t launchCrossMmaT(Instance* in, const EdgeRef* dEdges, int count, const double* rates,
                                   const double* weights, double* scratch, dim3 grid) {
    constexpr int Sp = 8 * NT;
    const size_t smem = sizeof(double) * (2 * 32 * (size_t)(Sp + 4) + 32);
    k_cross_mma<NT><<<grid, 128, smem, in->stream>>>(dEdges, count, rates, weights, in->dPatternWeights, in->S, in->C,
                                                     in->P, in->Ppad, scratch);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
k_cross_reduce(const double* __restrict__ scratch, int nBlocks, int n, double* __restrict__ out) {
    const int q = blockIdx.x * 256 + threadIdx.x;
    if (q >= n) return;
    double v = 0.0;
    for (int b = 0; b < nBlocks; ++b) v += scratch[(size_t)b * n + q];
    out[q] = v;
}

// scratch must hold crossProductBlocks() * S * S + S * S doubles; the result lands in the last S * S.
static void crossGeometry(const Instance* in, int count, int& pch, int& chunks, int& groups, bool& mma) {
    const bool four = in->Sp == 4 && in->S == 4;        // k_cross4 writes S x S = 16 entries per block
    const int nt = in->Sp / 8;
    mma = !four && in->genericMma && in->Sp % 8 == 0 && ((nt >= 1 && nt <= 4) || nt == 8);
    pch = four ? 256 : (mma ? 32 : std::max(1, std::min(32, 2048 / in->S)));
    chunks = (in->P + pch - 1) / pch;
    // the tensor form is a chain of short dependent phases per edge: fill every SM with 4 resident blocks
    // (whole blocks per wave only: a partial second wave would double the run time of this latency-chained kernel)
    groups = mma ? std::max(1, std::min(count, 4 * in->smCount / chunks))
                 : std::max(1, std::min(count, ((four ? 4 : 2) * in->smCount + chunks - 1) / chunks));
}

int crossProductBlocks(const Instance* in, int count) {
    int pch, chunks, groups; bool mma;
    crossGeometry(in, count, pch, chunks, groups, mma);
    return chunks * groups;
}

cudaError_t launchCrossProducts(Instance* in, const EdgeRefT<void>* dRefs, int count, const double* rates,
                                const double* weights, double* scratch) {
    const EdgeRef* dEdges = reinterpret_cast<const EdgeRef*>(dRefs);
    const EdgeRefT<float>* dEdgesF = reinterpret_cast<const EdgeRefT<float>*>(dRefs);
    int pch, chunks, groups; bool mma;
    crossGeometry(in, count, pch, chunks, groups, mma);
    const int n = in->S * in->S;
    dim3 grid(chunks, groups);
    cudaError_t e = cudaSuccess;
    if (in->Sp == 4 && in->S == 4) {
        if (in->single)
            k_cross4_f32<<<grid, 256, 0, in->stream>>>(dEdgesF, count, rates, weights, in->dPatternWeights, in->C, in->P,
                                                       in->Ppad, scratch);
        else
            k_cross4<<<grid, 256, 0, in->stream>>>(dEdges, count, rates, weights, in->dPatternWeights, in->C, in->P,
                                                   in->Ppad, scratch);
        e = cudaGetLastError();
    } else if (mma) {
        switch (in->Sp / 8) {
            case 1: e = launchCrossMmaT<1>(in, dEdges, count, rates, weights, scratch, grid); break;
            case 2: e = launchCrossMmaT<2>(in, dEdges, count, rates, weights, scratch, grid); break;
            case 3: e = launchCrossMmaT<3>(in, dEdges, count, rates, weights, scratch, grid); break;
            case 4: e = launchCrossMmaT<4>(in, dEdges, count, rates, weights, scratch, grid); break;
            default: e = launchCrossMmaT<8>(in, dEdges, count, rates, weights, scratch, grid); break;
        }
    } else {
        const int S4 = (in->S + 3) & ~3;
        const size_t smem = sizeof(double) * ((size_t)((pch + 1) & ~1) + 2 * (size_t)pch * S4);
        if (smem > 48 * 1024) {
            e = cudaFuncSetAttribute(k_cross_generic, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
        }
        if (in->single)
            k_cross_generic_f32<<<grid, 256, smem, in->stream>>>(dEdgesF, count, rates, weights, in->dPatternWeights, in->S,
                                                                 in->Sp, in->C, in->P, in->Ppad, pch, scratch);
        else
            k_cross_generic<<<grid, 256, smem, in->stream>>>(dEdges, count, rates, weights, in->dPatternWeights, in->S,
                                                             in->Sp, in->C, in->P, in->Ppad, pch, scratch);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) return e;
    k_cross_reduce<<<(n + 255) / 256, 256, 0, in->stream>>>(scratch, chunks * groups, n,
                                                            scratch + (size_t)chunks * groups * n);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// root integration + reduction
// ---------------------------------------------------------------------------------------------
// site[p] = log(sum_i pi_i (sum_c w_c root[c,p,i])) + cum[p]   (GeneralLikelihoodCore.java:358-408)
// out     = sum_p weight[p] site[p], deterministic two-level tree (fixed shape => reproducible).
__device__ __forceinline__ void storeSys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long loadSys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// Called by one whole block (>= size threads, all of them): stores `mine` into every member's slot array, waits for the
// others' entries of this evaluation on the own device and leaves out[0] = sum in rank order, out[1] = mine.
__device__ __forceinline__ void exchangeJoint(const Exchange& ex, double mine, double* __restrict__ out) {
    __shared__ double theirs[kMaxGroup];
    const int bank = (int)(ex.seq & 1ull);
    if ((int)threadIdx.x < ex.size) {
        const int q = threadIdx.x;
        ExchangeSlot* dst = ex.peers[q] + bank * ex.size + ex.rank;
        dst->value = mine;
        __threadfence_system();
        storeSys(&dst->seq, ex.seq);
        const ExchangeSlot* src = ex.peers[ex.rank] + bank * ex.size + q;         // own device's copy of member q's entry
        const long long t0 = clock64();
        bool ok = true;
        while (loadSys(&src->seq) != ex.seq) {
            if (clock64() - t0 > ex.timeoutCycles) { ok = false; break; }
            __nanosleep(64);
        }
        theirs[q] = ok ? src->value : __longlong_as_double(0x7ff8000000000000ll);   // a peer never arrived: NaN
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double joint = 0.0;
        for (int q = 0; q < ex.size; ++q) joint += theirs[q];                     // rank order: identical on every member
        out[0] = joint;
        out[1] = mine;
    }
}

template <typename T>
__device__ __forceinline__ void rootBody(const T* __restrict__ root, const double* __restrict__ weights,
                                         const double* __restrict__ freqs, const double* __restrict__ cumScale,
                                         const double* __restrict__ patternWeights, int S, int Sp, int C, int Ppad, int pBegin,
                                         int pEnd, double* __restrict__ site, double* __restrict__ blockSums,
                                         unsigned int* __restrict__ counter, double* __restrict__ out, const Exchange& ex) {
    __shared__ double red[256];
    __shared__ bool last;
    const int p = pBegin + blockIdx.x * blockDim.x + threadIdx.x;
    double contrib = 0.0;
    if (p < pEnd) {
        double sum = 0.0;
        for (int i = 0; i < S; ++i) {
            double integ = 0.0;
            for (int c = 0; c < C; ++c) integ += root[((size_t)c * Ppad + p) * Sp + i] * weights[c];
            sum += freqs[i] * integ;
        }
        double s = log(sum);
        if (cumScale != nullptr) s += cumScale[p];
        site[p] = s;
        contrib = patternWeights[p] * s;
    }
    red[threadIdx.x] = contrib;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        blockSums[blockIdx.x] = red[0];
        __threadfence();
        unsigned int done = atomicAdd(counter, 1u);
        last = (done == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        __threadfence();
        double acc = 0.0;
        for (int q = threadIdx.x; q < (int)gridDim.x; q += blockDim.x) acc += blockSums[q];
        red[threadIdx.x] = acc;
        __syncthreads();
        for (int w = 128; w > 0; w >>= 1) {
            if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
            __syncthreads();
        }
        if (ex.size <= 1) {
            if (threadIdx.x == 0) { *out = red[0]; *counter = 0u; }
            return;
        }
        // ---- reduce group: this shard's sum goes to every member over NVLink, theirs are added here (engine.h, Exchange)
        exchangeJoint(ex, red[0], out);
        if (threadIdx.x == 0) *counter = 0u;
    }
}

__global__ void __launch_bounds__(256)
k_root(const double* __restrict__ root, const double* __restrict__ weights, const double* __restrict__ freqs,
       const double* __restrict__ cumScale, const double* __restrict__ patternWeights, int S, int Sp, int C,
       int Ppad, int pBegin, int pEnd, double* __restrict__ site, double* __restrict__ blockSums,
       unsigned int* __restrict__ counter, double* __restrict__ out, const Exchange ex) {
    rootBody(root, weights, freqs, cumScale, patternWeights, S, Sp, C, Ppad, pBegin, pEnd, site, blockSums, counter, out, ex);
}

__global__ void __launch_bounds__(256)
k_root_f32(const float* __restrict__ root, const double* __restrict__ weights, const double* __restrict__ freqs,
           const double* __restrict__ cumScale, const double* __restrict__ patternWeights, int S, int Sp, int C,
           int Ppad, int pBegin, int pEnd, double* __restrict__ site, double* __restrict__ blockSums,
           unsigned int* __restrict__ counter, double* __restrict__ out, const Exchange ex) {
    rootBody(root, weights, freqs, cumScale, patternWeights, S, Sp, C, Ppad, pBegin, pEnd, site, blockSums, counter, out, ex);
}

// sum of `n` device values (the per-partition sums of a *ByPartition root call), then the same exchange: one block
__global__ void __launch_bounds__(64)
k_exchange_sum(const double* __restrict__ vals, int n, double* __restrict__ out, const Exchange ex) {
    __shared__ double mine;
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int k = 0; k < n; ++k) s += vals[k];
        mine = s;
    }
    __syncthreads();
    exchangeJoint(ex, mine, out);
}

cudaError_t launchExchangeSum(Instance* in, const double* dVals, int n, double* dOutJoint, const Exchange* exchange) {
    k_exchange_sum<<<1, 64, 0, in->stream>>>(dVals, n, dOutJoint, *exchange);
    return cudaGetLastError();
}

cudaError_t launchRoot(Instance* in, const void* root, const double* weights, const double* freqs,
                       const double* cumScale, int pBegin, int pEnd, double* dOutSlot, const Exchange* exchange) {
    int n = pEnd - pBegin;
    Exchange ex;                       // size 1: no exchange
    if (exchange != nullptr) ex = *exchange;
    if (n <= 0 && ex.size <= 1) return cudaMemsetAsync(dOutSlot, 0, sizeof(double), in->stream);
    int blocks = std::max(1, (n + 255) / 256);       // an empty shard still takes part in the exchange (sum 0)
    if (in->single)
        k_root_f32<<<blocks, 256, 0, in->stream>>>(static_cast<const float*>(root), weights, freqs, cumScale,
                                                   in->dPatternWeights, in->S, in->Sp, in->C, in->Ppad, pBegin, pEnd,
                                                   in->dSite, in->dBlockSums, in->dCounter, dOutSlot, ex);
    else
        k_root<<<blocks, 256, 0, in->stream>>>(static_cast<const double*>(root), weights, freqs, cumScale,
                                               in->dPatternWeights, in->S, in->Sp, in->C, in->Ppad, pBegin, pEnd,
                                               in->dSite, in->dBlockSums, in->dCounter, dOutSlot, ex);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// scale-factor accumulation:  cum[p] += sign * sum_k log-factor_k[p]   (BDLD:915-926)
// ---------------------------------------------------------------------------------------------
// block = 32 patterns x 16 buffer-lanes: lane j sums buffers j, j+16, ... (independent loads in flight), then a
// fixed-order reduction over the 16 lanes -> deterministic, and N-1 buffers no longer serialise on one thread.
__global__ void __launch_bounds__(512)
k_scale_accum(const double* __restrict__ scaleBase, int Ppad, const int* __restrict__ idx,
              int count, double* __restrict__ cum, double sign, int logScalers, int pBegin, int pEnd) {
    __shared__ double part[16][33];
    const int px = threadIdx.x, ky = threadIdx.y;
    const int p = pBegin + blockIdx.x * 32 + px;
    double acc = 0.0;
    if (p < pEnd) {
#pragma unroll 4
        for (int k = ky; k < count; k += 16) {
            const double f = scaleBase[(size_t)idx[k] * Ppad + p];
            acc += logScalers ? f : log(f);
        }
    }
    part[ky][px] = acc;
    __syncthreads();
    if (ky == 0 && p < pEnd) {
        double s = 0.0;
#pragma unroll
        for (int j = 0; j < 16; ++j) s += part[j][px];
        cum[p] += sign * s;
    }
}

cudaError_t launchScaleAccumulate(Instance* in, const int* dIdx, int count, double* cum, double sign,
                                  int pBegin, int pEnd) {
    int n = pEnd - pBegin;
    if (n <= 0 || count <= 0) return cudaSuccess;
    k_scale_accum<<<(n + 31) / 32, dim3(32, 16), 0, in->stream>>>(in->dScale, in->Ppad, dIdx, count, cum, sign,
                                                                  in->logScalers ? 1 : 0, pBegin, pEnd);
    return cudaGetLastError();
}

// getPartials with a cumulative scale index: tmp[c,p,i] *= exp(cum[p])
__global__ void k_unscale(double* __restrict__ tmp, const double* __restrict__ cum, int Sp, int Ppad, size_t n) {
    size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    int p = (int)((q / Sp) % Ppad);
    tmp[q] *= exp(cum[p]);
}

cudaError_t launchRescalePartialsForGet(Instance* in, double* tmp, const double* cum) {
    size_t n = in->partialsElems;
    k_unscale<<<(unsigned)((n + 255) / 256), 256, 0, in->stream>>>(tmp, cum, in->Sp, in->Ppad, n);
    return cudaGetLastError();
}

}  // namespace b200
