// ancestral.cu -- joint ancestral-state sampling on the device (b200SampleAncestralStates, DESIGN.md §7).
//
// Per pattern p the kernels draw ONE sample of (rate category, state of every listed node) from the exact joint posterior
// given the tip data, the post-order partials the instance holds and its transition matrices:
//   root row : (c, i) with probability ∝ w_c · π_i · Lroot_c[p][i]
//   row r    : j given the parent row's state i and the root's category c, ∝ P_c[i][j] · L_r,c[p][j]
//              (a compact tip keeps its observed state; a gap / unknown state (>= S) draws ∝ P_c[i][j])
// Rows arrive in pre-order (every parent before its children) and one thread (4-state matrix layout) or one warp (generic
// layout) per pattern walks them in that order; a parent's state comes from registers when it is the previous row, else
// from the output the same thread (warp) wrote earlier.  Per-pattern rescale factors cancel in every conditional, so scale
// buffers are not read.  No atomics: the output is a pure function of the inputs, seed and draw index.
//
// Uniforms: Philox4x64-10 (the generator of numpy.random.Philox), key (seed, 0), counter (drawIndex, global pattern, row, 0);
// the first output word x gives u = (x >> 11) · 2^-53.  The draw is an inverse CDF over the items in index order ((c, i)
// c-major at the root) with fp64 cumulative sums: the first item whose cumulative sum exceeds u · total.  If none does
// (total zero or not finite: data impossible under the model; or rounding at the top end) the last item of positive weight
// is taken, and item 0 when there is none.
//
// Markov jumps (b200SampleMarkovJumps, DESIGN.md §7.2): the same kernels, instantiated with Jumps = true, draw exactly the
// same sample and look up, per drawn branch pair (i -> j), the conditional expectation N_g,c,r[i][j] of every register g
// that k_jump_conditional wrote beforehand.  Pattern totals stay in registers; per-(row, pattern) values go to a
// [g][row][P] workspace that k_jump_branch_totals reduces in a fixed order.
#include "walk4.cuh"

#include <algorithm>

namespace b200 {

namespace {

__host__ __device__ __forceinline__ uint64_t mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// first 64-bit word of the Philox4x64-10 block at counter (c0, c1, c2, c3) under key (k0, k1) (Salmon et al., SC'11)
__host__ __device__ __forceinline__ uint64_t philox4x64_10(uint64_t k0, uint64_t k1, uint64_t c0, uint64_t c1, uint64_t c2, uint64_t c3) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
        const uint64_t lo0 = 0xD2E7470EE14C6C93ull * c0, hi0 = mulhi64(0xD2E7470EE14C6C93ull, c0);
        const uint64_t lo1 = 0xCA5A826395121157ull * c2, hi1 = mulhi64(0xCA5A826395121157ull, c2);
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    }
    return c0;
}

__device__ __forceinline__ double uniformAt(const AncestralArgs& a, int p, int row) {
    const uint64_t x = philox4x64_10(a.seed, 0, a.drawIndex, (uint64_t)(a.pOffset + p), (uint64_t)row, 0);
    return (double)(x >> 11) * 0x1.0p-53;
}

// ---- S <= 4, matrices [j][CP][i]: one thread per pattern ------------------------------------------------------------------
// L of a row in category c: its partials cell, or the indicator of a compact tip's state (all ones for a gap)
template <typename T>
__device__ __forceinline__ void cell4(const AncestralArgs& a, int4 row, int c, int p, double (&L)[4]) {
    if (row.x >= 0) {
        loadCell(static_cast<const T*>(a.partials) + (size_t)row.x * a.stride + ((size_t)c * a.Ppad + p) * 4, L);
    } else {
        const int s = a.states8[(size_t)(-row.x - 1) * a.Ppad + p];
#pragma unroll
        for (int j = 0; j < 4; ++j) L[j] = (s >= a.S || s == j) ? 1.0 : 0.0;
    }
}

// Markov jumps: n_g of the branch above row r for the drawn pair (i -> j) in category c, looked up in N [g][row][C][S][S]
__device__ __forceinline__ const double* jumpCell(const AncestralArgs& a, const MarkovJumpArgs& mj, int r, int c, int i, int j) {
    return mj.cond + (((size_t)r * a.C + c) * a.S + i) * a.S + j;
}

template <typename T, bool Jumps>
__global__ void __launch_bounds__(64)
k_ancestral4(const AncestralArgs a, const MarkovJumpArgs mj) {
    const int p = blockIdx.x * 64 + threadIdx.x;
    if (p >= a.P) return;
    const int S = a.S;
    double total_g[Jumps ? kMaxJumpRegisters : 1] = {};  // pattern totals, summed in row order
    // root: (c, i) jointly, two passes over the same products so that the running sum reproduces the total exactly
    const int4 root = __ldg(a.rows);
    double total = 0.0;
    for (int c = 0; c < a.C; ++c) {
        double L[4];
        cell4<T>(a, root, c, p, L);
        const double wc = a.weights[c];
#pragma unroll
        for (int i = 0; i < 4; ++i) if (i < S) total += wc * a.freqs[i] * L[i];
    }
    const double t0 = uniformAt(a, p, 0) * total;
    int pick = -1, last = 0;
    double cum = 0.0;
    for (int c = 0; c < a.C && pick < 0; ++c) {
        double L[4];
        cell4<T>(a, root, c, p, L);
        const double wc = a.weights[c];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (i >= S || pick >= 0) continue;
            const double w = wc * a.freqs[i] * L[i];
            cum += w;
            if (w > 0.0) last = c * S + i;
            if (t0 < cum) pick = c * S + i;
        }
    }
    if (pick < 0) pick = last;
    const int cat = pick / S;
    int prev = pick % S;
    a.outCategories[p] = cat;
    a.outStates[p] = prev;
    for (int r = 1; r < a.count; ++r) {
        const int4 row = __ldg(a.rows + r);
        const int i = row.y == r - 1 ? prev : a.outStates[(size_t)row.y * a.P + p];
        int j;
        const int tipState = row.x < 0 ? a.states8[(size_t)(-row.x - 1) * a.Ppad + p] : S;
        if (tipState < S) {
            j = tipState;
        } else {
            double L[4];
            cell4<T>(a, row, cat, p, L);
            const double* m = a.mats + (size_t)row.z * a.matStride + (size_t)cat * 4 + i;     // P_c[i][j] at [j][CP][i]
            double w[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) w[q] = q < S ? __ldg(m + (size_t)q * a.CP * 4) * L[q] : 0.0;
            double tot = 0.0;
#pragma unroll
            for (int q = 0; q < 4; ++q) tot += w[q];
            const double t = uniformAt(a, p, r) * tot;
            j = -1;
            int lastPos = 0;
            double run = 0.0;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                run += w[q];
                if (w[q] > 0.0) lastPos = q;
                if (j < 0 && q < S && t < run) j = q;
            }
            if (j < 0) j = lastPos;
        }
        a.outStates[(size_t)r * a.P + p] = j;
        if constexpr (Jumps) {
            const double* n = jumpCell(a, mj, r, cat, i, j);
            const size_t gStride = (size_t)a.count * a.C * S * S;
#pragma unroll
            for (int g = 0; g < kMaxJumpRegisters; ++g) {
                if (g >= mj.G) break;
                const double v = __ldg(n + g * gStride);
                total_g[g] += v;
                if (mj.perRow != nullptr) mj.perRow[((size_t)g * a.count + r) * a.P + p] = v;
            }
        }
        prev = j;
    }
    if constexpr (Jumps) {
        if (mj.pattern != nullptr) {
#pragma unroll
            for (int g = 0; g < kMaxJumpRegisters; ++g) if (g < mj.G) mj.pattern[(size_t)g * a.P + p] = total_g[g];
        }
    }
}

// ---- generic layout (S > 4, or C > 32): one warp per pattern, lanes over the items, shuffle prefix sums -----------------
// item q of n drawn ∝ weight(q); every lane returns the same index
template <typename F>
__device__ __forceinline__ int drawWarp(int n, double u, const F& weight) {
    const int lane = threadIdx.x & 31;
    double total = 0.0;
    for (int base = 0; base < n; base += 32) {
        double w = base + lane < n ? weight(base + lane) : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
        total += w;
    }
    const double t = u * total;
    double carry = 0.0;
    int last = 0, found = -1;
    for (int base = 0; base < n && found < 0; base += 32) {
        const int q = base + lane;
        const double w = q < n ? weight(q) : 0.0;
        double x = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        const unsigned hit = __ballot_sync(0xffffffffu, q < n && t < carry + x);
        const unsigned pos = __ballot_sync(0xffffffffu, w > 0.0);
        if (hit) found = base + __ffs(hit) - 1;
        if (pos) last = base + 31 - __clz((int)pos);
        carry += __shfl_sync(0xffffffffu, x, 31);
    }
    return found >= 0 ? found : last;
}

// Markov jumps: lane g < G follows register g
template <bool Jumps>
__global__ void __launch_bounds__(128)
k_ancestral_warp(const AncestralArgs a, const MarkovJumpArgs mj) {
    const int p = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (p >= a.P) return;                                   // warp-uniform
    const int lane = threadIdx.x & 31, S = a.S, Sp = a.Sp;
    double total = 0.0;                                     // Markov jumps: lane g's pattern total, in row order
    const double* part = static_cast<const double*>(a.partials);
    auto L = [&](int4 row, int c, int j) -> double {
        if (row.x >= 0) return part[(size_t)row.x * a.stride + ((size_t)c * a.Ppad + p) * Sp + j];
        const int s = a.states32[(size_t)(-row.x - 1) * a.Ppad + p];
        return (s >= S || s == j) ? 1.0 : 0.0;
    };
    const int4 root = __ldg(a.rows);
    const int pick = drawWarp(a.C * S, uniformAt(a, p, 0), [&](int q) {
        const int c = q / S, i = q - c * S;
        return a.weights[c] * a.freqs[i] * L(root, c, i);
    });
    const int cat = pick / S;
    int prev = pick - cat * S;
    if (lane == 0) { a.outCategories[p] = cat; a.outStates[p] = prev; }
    for (int r = 1; r < a.count; ++r) {
        const int4 row = __ldg(a.rows + r);
        __syncwarp();                                       // lane 0's earlier stores are visible to the whole warp
        const int i = row.y == r - 1 ? prev : a.outStates[(size_t)row.y * a.P + p];
        const int tipState = row.x < 0 ? a.states32[(size_t)(-row.x - 1) * a.Ppad + p] : S;
        // an observed tip state draws over no items (no branch around the shuffles: ptxas then keeps no convergence state)
        const double* m = a.mats + (size_t)row.z * a.matStride + (size_t)cat * Sp * Sp + i;       // P_c[i][j] at MT[c][j][i]
        const int drawn = drawWarp(tipState < S ? 0 : S, uniformAt(a, p, r),
                                   [&](int q) { return m[(size_t)q * Sp] * L(row, cat, q); });
        const int j = tipState < S ? tipState : drawn;
        if (lane == 0) a.outStates[(size_t)r * a.P + p] = j;
        if constexpr (Jumps) {
            if (lane < mj.G) {
                const double v = __ldg(jumpCell(a, mj, r, cat, i, j) + (size_t)lane * a.count * a.C * S * S);
                total += v;
                if (mj.perRow != nullptr) mj.perRow[((size_t)lane * a.count + r) * a.P + p] = v;
            }
        }
        prev = j;
    }
    if constexpr (Jumps) {
        if (mj.pattern != nullptr && lane < mj.G) mj.pattern[(size_t)lane * a.P + p] = total;
    }
}

// ---- Markov jumps (b200SampleMarkovJumps, DESIGN.md §7.2) -------------------------------------------------------------------
// With Q = V diag(λ) V^-1 and a register matrix M_g, the expected register total along a branch of time τ jointly with its
// end state is E = V (W_g ∘ I(τ)) V^-1, W_g = V^-1 M_g V, I_kl(τ) = τ e^{λ_l τ} φ((λ_k - λ_l) τ), φ(x) = expm1(x)/x;
// conditioned on the end points N = E / P̂ with P̂ = |V diag(e^{λτ}) V^-1| in the k_transition formula and order.
constexpr int kJumpPanel = 16;                              // output columns per pass of k_jump_conditional

__host__ __device__ constexpr size_t jumpSmemDoubles(int S) { return (size_t)S * S + S + 2 * (size_t)S * kJumpPanel; }

// W_g = V^-1 M_g V, once per call; grid (S, G): block (i, g) writes row i of W_g
__global__ void __launch_bounds__(128)
k_jump_registers(const MarkovJumpArgs m, int S) {
    extern __shared__ double y[];                           // [S]: row i of V^-1 M_g
    const int i = blockIdx.x, g = blockIdx.y;
    const double* V = m.eigen;
    const double* Vi = m.eigen + (size_t)S * S;
    const double* M = m.registers + (size_t)g * S * S;
    for (int l = threadIdx.x; l < S; l += blockDim.x) {
        double acc = 0.0;
        for (int q = 0; q < S; ++q) acc += Vi[(size_t)i * S + q] * M[(size_t)q * S + l];
        y[l] = acc;
    }
    __syncthreads();
    for (int l = threadIdx.x; l < S; l += blockDim.x) {
        double acc = 0.0;
        for (int q = 0; q < S; ++q) acc += y[q] * V[(size_t)q * S + l];
        m.W[((size_t)g * S + i) * S + l] = acc;
    }
}

// N of every register for one (row r >= 1, category c): grid (count - 1, C).  Shared memory: I [S][S], e^{λτ} [S], and per
// panel of kJumpPanel output columns P̂ and T = (W_g ∘ I) V^-1 [S][kJumpPanel]; P̂ is computed once per panel, then every
// register reuses it.  I_kl is evaluated with the larger of λ_k, λ_l in the exponential (the same value, by the symmetry of
// I): expm1 then never sees a positive argument and cannot overflow.
__global__ void __launch_bounds__(256)
k_jump_conditional(const MarkovJumpArgs m, int S, int C, int count) {
    extern __shared__ double sm[];
    double* I = sm;
    double* e = I + (size_t)S * S;
    double* Pp = e + S;
    double* T = Pp + (size_t)S * kJumpPanel;
    const int r = blockIdx.x + 1, c = blockIdx.y;
    const double* V = m.eigen;
    const double* Vi = m.eigen + (size_t)S * S;
    const double* lam = m.eigen + 2 * (size_t)S * S;
    const double tau = m.lengths[r] * m.rates[c];            // the product k_transition forms
    for (int k = threadIdx.x; k < S; k += blockDim.x) e[k] = exp(tau * lam[k]);
    __syncthreads();
    for (int idx = threadIdx.x; idx < S * S; idx += blockDim.x) {
        const int k = idx / S, l = idx - k * S;
        const double x = -fabs(lam[k] - lam[l]) * tau;
        const double phi = x == 0.0 ? 1.0 : expm1(x) / x;
        I[idx] = tau * e[lam[k] >= lam[l] ? k : l] * phi;
    }
    const size_t gStride = (size_t)count * C * S * S;
    double* out = m.cond + ((size_t)r * C + c) * S * S;
    for (int j0 = 0; j0 < S; j0 += kJumpPanel) {
        const int nj = min(kJumpPanel, S - j0);
        for (int idx = threadIdx.x; idx < S * nj; idx += blockDim.x) {
            const int i = idx / nj, jj = idx - i * nj, j = j0 + jj;
            double acc = 0.0;
            for (int k = 0; k < S; ++k) acc += V[(size_t)i * S + k] * (e[k] * Vi[(size_t)k * S + j]);
            Pp[i * kJumpPanel + jj] = fabs(acc);
        }
        for (int g = 0; g < m.G; ++g) {
            const double* W = m.W + (size_t)g * S * S;
            __syncthreads();                                // I, P̂ written; the previous register's T consumed
            for (int idx = threadIdx.x; idx < S * nj; idx += blockDim.x) {
                const int k = idx / nj, jj = idx - k * nj;
                double acc = 0.0;
                for (int l = 0; l < S; ++l) acc += (W[(size_t)k * S + l] * I[(size_t)k * S + l]) * Vi[(size_t)l * S + j0 + jj];
                T[k * kJumpPanel + jj] = acc;
            }
            __syncthreads();
            for (int idx = threadIdx.x; idx < S * nj; idx += blockDim.x) {
                const int i = idx / nj, jj = idx - i * nj;
                double E = 0.0;
                for (int k = 0; k < S; ++k) E += V[(size_t)i * S + k] * T[k * kJumpPanel + jj];
                const double ph = Pp[i * kJumpPanel + jj];
                out[(size_t)g * gStride + (size_t)i * S + j0 + jj] = ph > 0.0 ? E / ph : 0.0;
            }
        }
        __syncthreads();                                    // P̂ of this panel consumed
    }
}

// branch totals Σ_p w_p n_g[r][p]: grid (count, G), a fixed-order block reduction (no atomics; row 0 is 0)
__global__ void __launch_bounds__(256)
k_jump_branch_totals(const MarkovJumpArgs m, int count, int P) {
    __shared__ double red[256];
    const int r = blockIdx.x, g = blockIdx.y;
    double s = 0.0;
    if (r > 0) {
        const double* v = m.perRow + ((size_t)g * count + r) * P;
        for (int p = threadIdx.x; p < P; p += 256) s += m.patternWeights[p] * v[p];
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) m.branch[(size_t)g * count + r] = red[0];
}

}  // namespace

bool markovJumpsFit(const Instance* in) {
    return jumpSmemDoubles(in->S) * sizeof(double) <= std::max<size_t>(in->maxSmemOptin, 48 << 10);
}

cudaError_t launchMarkovJumps(Instance* in, const AncestralArgs& a, const MarkovJumpArgs& m) {
    const int S = in->S, C = in->C;
    k_jump_registers<<<dim3(S, m.G), S <= 32 ? 32 : 128, sizeof(double) * S, in->stream>>>(m, S);
    if (a.count > 1) {
        const size_t smem = jumpSmemDoubles(S) * sizeof(double);
        if (smem > (48 << 10)) {
            // the device's whole opt-in, never a smaller value: instances on other host threads launch the same kernel
            const cudaError_t e = cudaFuncSetAttribute(k_jump_conditional, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       (int)in->maxSmemOptin);
            if (e != cudaSuccess) return e;
        }
        const int work = S * std::min(S, kJumpPanel);
        const int threads = std::min(256, std::max(32, (work + 31) / 32 * 32));
        k_jump_conditional<<<dim3(a.count - 1, C), threads, smem, in->stream>>>(m, S, C, a.count);
    }
    const int blocks4 = (a.P + 63) / 64;
    if (in->matCP > 0) {
        if (in->single) k_ancestral4<float, true><<<blocks4, 64, 0, in->stream>>>(a, m);
        else k_ancestral4<double, true><<<blocks4, 64, 0, in->stream>>>(a, m);
    } else {
        k_ancestral_warp<true><<<(a.P + 3) / 4, 128, 0, in->stream>>>(a, m);
    }
    if (m.branch != nullptr) k_jump_branch_totals<<<dim3(a.count, m.G), 256, 0, in->stream>>>(m, a.count, a.P);
    return cudaGetLastError();
}

cudaError_t launchAncestral(Instance* in, const AncestralArgs& args) {
    if (in->matCP > 0) {
        const int blocks = (args.P + 63) / 64;
        if (in->single) k_ancestral4<float, false><<<blocks, 64, 0, in->stream>>>(args, MarkovJumpArgs{});
        else k_ancestral4<double, false><<<blocks, 64, 0, in->stream>>>(args, MarkovJumpArgs{});
    } else {
        k_ancestral_warp<false><<<(args.P + 3) / 4, 128, 0, in->stream>>>(args, MarkovJumpArgs{});
    }
    return cudaGetLastError();
}

}  // namespace b200
