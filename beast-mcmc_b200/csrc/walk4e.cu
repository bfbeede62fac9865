// walk4e.cu -- the 4-state (nucleotide) walk in EIGEN FORM: the default updatePartials kernel of S <= 4 instances.
//
// What bounds k_walk4: the L1/LSU data pipe, most of it matrix traffic -- every thread needs its category's 4x4 matrix in
// registers (128 B per child)
// and a compact-tip child costs one 32-B matrix column per PATTERN -- while HBM only saw the mandatory destination writes.
//
// Here no transition matrix is read at all.  With one real eigen system per list (what HomogenousSubstitutionModelDelegate
// hands over, HSMD:228-266)
//        P_c(t) x = V ( e ⊙ (V^-1 x) ),     e_k = exp(lambda_k r_c t)
// so a branch is 4 doubles per category ("spectrum", written by k_transition4 next to the matrices) and V, V^-1 are the same
// for every op of the launch: they travel BY VALUE in the kernel parameters, i.e. in the constant bank, and reach the FP64
// pipe as uniform-register operands (SASS: LDCU.128 + DFMA R, R, UR, R) -- zero registers, zero LSU wavefronts.
//   internal child : u = V^-1 x (16 FMA), w = e ⊙ u (4), y = |V w| (16)        -- 32 B of spectrum instead of 128 B of matrix
//   compact tip    : u_k = V^-1[k][s] (register selects on the state byte), then as above; gap/unknown -> y = 1
// |.| mirrors the reference's abs() on P(t) entries (BaseSubstitutionModel.java:236): for a tip the value IS |P[i][s]|
// with the reference's own summation order; partials stay non-negative.  The FP64 pipe goes from 12 % to ~40 % busy; the
// LSU data pipe keeps only what is irreducible: destination stores, the child cells that are not forwarded in registers,
// spectra, op records.  Lists the form does not cover (matrices set directly or convolved, complex pairs, several eigen
// systems in one list) run on k_walk4; pre-order lists keep their own kernel.  Results agree with the matrix form to
// rounding (tests/test_gpu_parity.py::test_walk_variants_agree, 1e-13).
//
// ALIGNED = every op spans whole 32-pattern groups [0, Ppad): no per-pattern predicates at all (padded columns hold
// harmless finite values and are never read back).  Partition windows take the predicated instance.
#include <atomic>
#include <cstdio>

#include "engine.h"
#include "walk4.cuh"

namespace b200 {

namespace {

// Compact-tip children: at CP <= 8 (TABLE) the columns of P for the five possible tip symbols (4 states + gap) of all
// categories are staged once per (op, child) in a per-warp shared-memory table by a handful of lanes; every pattern then
// picks its 32-B column with two LDS.128 -- no FP64 work, no dependent global load.  At CP = 16 and 32 a tip goes through
// the same contraction as an internal child, with a one-hot x (no memory traffic, no extra code path).
__device__ __forceinline__ double absBits(double v) {       // |v| on the integer pipe (the FP64 pipe is the busy one here)
    return __hiloint2double(__double2hiint(v) & 0x7fffffff, __double2loint(v));
}

template <typename T, int CP, int R, bool ALIGNED, bool FIRST>
__device__ __forceinline__ void childTermE(const WalkArgs& A, const double (&Vi)[16], int child, int matIdx, bool fromRegisters,
                                           int cc, size_t off0, int p0, bool catValid, int pBegin, int pEnd, double (&d)[R][4],
                                           double* tab) {
    constexpr int G = 32 / CP;
    constexpr bool TABLE = CP <= 8;
    const int S = A.S;
    const bool tip = child < 0;
    if (TABLE && tip) {
        const int lane = threadIdx.x & 31;
        const uint8_t* t = A.states + (size_t)(-child - 1) * A.Ppad;
        int s[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int p = p0 + r * G;
            s[r] = (ALIGNED || (catValid && p >= pBegin && p < pEnd)) ? (int)__ldg(t + p) : 4;
        }
        // table [CP][5][4]: column s of P_c (the tip's contribution when it shows state s), s = 4 (and s >= S): all ones
        const double* m = A.mats + (size_t)matIdx * A.matStride;
        __syncwarp();                                              // the previous table of this slot is no longer read
#pragma unroll
        for (int q = lane; q < 5 * CP; q += 32) {
            const int c = q / 5, sym = q - 5 * c;
            double v[4];
            if (sym < S && sym < 4 && c < A.C) ldg256_ro(m + (sym * CP + c) * 4, v);
            else {
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = (i < S) ? 1.0 : 0.0;
            }
            double2* dst = reinterpret_cast<double2*>(tab + q * 4);
            dst[0] = make_double2(v[0], v[1]);
            dst[1] = make_double2(v[2], v[3]);
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const double2* col = reinterpret_cast<const double2*>(tab + (cc * 5 + min(s[r], 4)) * 4);
            const double2 lo = col[0], hi = col[1];
            if (FIRST) { d[r][0] = lo.x; d[r][1] = lo.y; d[r][2] = hi.x; d[r][3] = hi.y; }
            else { d[r][0] *= lo.x; d[r][1] *= lo.y; d[r][2] *= hi.x; d[r][3] *= hi.y; }
        }
        return;
    }
    double e[4];
    ldg256_ro(A.evecs + ((size_t)matIdx * CP + cc) * 4, e);
    const uint8_t* t = A.states + (size_t)(tip ? -child - 1 : 0) * A.Ppad;
    const T* xg = static_cast<const T*>(A.partials) + (size_t)(tip ? 0 : child) * A.stride + off0;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int p = p0 + r * G;
        const bool live = ALIGNED || (catValid && p >= pBegin && p < pEnd);
        double x[4], u[4], y[4];
        int s = 0;
        if (tip) {
            s = live ? (int)__ldg(t + p) : S;
#pragma unroll
            for (int j = 0; j < 4; ++j) x[j] = (s == j) ? 1.0 : 0.0;
        } else if (fromRegisters) {
#pragma unroll
            for (int i = 0; i < 4; ++i) x[i] = d[r][i];
        } else if (live) {
            loadCell(xg + (size_t)r * G * 4, x);
        } else {
            x[0] = x[1] = x[2] = x[3] = 0.0;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
            u[k] = (Vi[4 * k] * x[0] + Vi[4 * k + 1] * x[1] + Vi[4 * k + 2] * x[2] + Vi[4 * k + 3] * x[3]) * e[k];
#pragma unroll
        for (int i = 0; i < 4; ++i)
            y[i] = absBits(A.V[4 * i] * u[0] + A.V[4 * i + 1] * u[1] + A.V[4 * i + 2] * u[2] + A.V[4 * i + 3] * u[3]);
        if (tip && s >= S) {                                       // gap / unknown: every state is compatible
#pragma unroll
            for (int i = 0; i < 4; ++i) y[i] = (i < S) ? 1.0 : 0.0;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) d[r][i] = FIRST ? y[i] : d[r][i] * y[i];
    }
}

template <typename T, int CP, int R, bool ALIGNED>
__device__ __forceinline__ void walk4eBody(const WalkArgs& A) {
    constexpr int G = 32 / CP;
    constexpr bool TABLE = CP <= 8;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int c = lane / G;
    const int4 range = __ldg(A.subs + blockIdx.y);
    const int p0 = range.z + warp * (G * R) + (lane % G);          // patterns p0 + r*G
    if (range.z + warp * (G * R) >= range.w) return;               // whole warp outside this subtree's pattern window
    const bool catValid = c < A.C;
    const int cc = catValid ? c : 0;
    const size_t off0 = ((size_t)cc * A.Ppad + p0) * 4;
    const int last = range.y - 1;
    // per-warp tip tables: [child slot][CP][5][4] doubles
    __shared__ __align__(16) double tipTab[TABLE ? 4 * 2 * CP * 20 : 2];
    double* tab1 = tipTab + (TABLE ? ((threadIdx.x >> 5) * 2) * CP * 20 : 0);
    double* tab2 = tab1 + (TABLE ? CP * 20 : 0);

    // V^-1 in vector registers (the tip selects and the first contraction read it), V stays in the constant bank: both in
    // uniform registers do not fit (64 > 63) and ptxas would spill.  The asm keeps ptxas from folding the copy back.
    double Vi[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) asm volatile("mov.f64 %0, %1;" : "=d"(Vi[q]) : "d"(A.Vi[q]));
    Op4 cur = loadOp(A.ops + range.x);
    double d[R][4];                                                // survives the loop: op k+1 may take it as its first child
#pragma unroll
    for (int r = 0; r < R; ++r) d[r][0] = d[r][1] = d[r][2] = d[r][3] = 0.0;
    for (int k = range.x; k <= last; ++k) {
        Op4 nxt;
        if (R == 1) nxt = loadOp(A.ops + min(k + 1, last));
        else if (lane == 0) prefetchL1(A.ops + min(k + 2, last));
        // look-ahead: what the NEXT op reads from memory (never this op's destination) starts its trip to L1 now
#pragma unroll
        for (int w = 0; w < 2; ++w) {
            const int pf = w == 0 ? cur.pfA : cur.pfB;
            if (pf == 0) continue;
            if (pf & 1) {
                const uint8_t* t = A.states + (size_t)(pf >> 1) * A.Ppad + p0;
                if ((lane % G) == 0 && c == 0) prefetchL1(t);                  // G*R consecutive bytes: one line
            } else if (catValid) {
                const T* xg = static_cast<const T*>(A.partials) + (size_t)((pf >> 1) - 1) * A.stride + off0;
#pragma unroll
                for (int r = 0; r < R; ++r)
                    if (ALIGNED || p0 + r * G < A.Ppad) prefetchL1(xg + (size_t)r * G * 4);
            }
        }
        if (lane < 2) {
            const int mi = lane == 0 ? cur.pfM1 : cur.pfM2;
            if (mi >= 0) prefetchL1(A.evecs + (size_t)mi * CP * 4);            // all categories of a branch: one 128-B line
        } else if (TABLE && lane >= 8 && lane < 16) {
            const int mi = lane < 12 ? cur.pfM1 : cur.pfM2;                     // matrix rows, should a child be a compact tip
            if (mi >= 0) prefetchL1(A.mats + (size_t)mi * A.matStride + (lane & 3) * 4 * CP);
        }
        childTermE<T, CP, R, ALIGNED, true>(A, Vi, cur.c1, cur.m1, (cur.pad_ & 2) != 0, cc, off0, p0, catValid, cur.pBegin, cur.pEnd, d, tab1);
        childTermE<T, CP, R, ALIGNED, false>(A, Vi, cur.c2, cur.m2, false, cc, off0, p0, catValid, cur.pBegin, cur.pEnd, d, tab2);
        if (R != 1) nxt = loadOp(A.ops + min(k + 1, last));
        T* dg = static_cast<T*>(A.partials) + (size_t)cur.dest * A.stride + off0;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int p = p0 + r * G;
            const bool active = ALIGNED ? catValid : (catValid && p >= cur.pBegin && p < cur.pEnd);
            // ---- rescaling (AbstractLikelihoodCore.java:406-442, unconditional as in BEAGLE) -----
            if (cur.sw >= 0) {
                double m = active ? fmax(fmax(d[r][0], d[r][1]), fmax(d[r][2], d[r][3])) : 0.0;
#pragma unroll
                for (int sh = G; sh < 32; sh <<= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, sh));
                if (m == 0.0) m = 1.0;
                const double inv = 1.0 / m;
#pragma unroll
                for (int i = 0; i < 4; ++i) d[r][i] *= inv;
                if (active && c == 0) A.scale[(size_t)cur.sw * A.Ppad + p] = A.logScalers ? log(m) : m;
            } else if (cur.sr >= 0) {
                double f = active ? A.scale[(size_t)cur.sr * A.Ppad + p] : 1.0;
                if (A.logScalers) f = exp(f);
                const double inv = 1.0 / f;
#pragma unroll
                for (int i = 0; i < 4; ++i) d[r][i] *= inv;
            }
            roundCell<T>(d[r]);
            if (active) storeCell(dg + (size_t)r * G * 4, d[r]);
        }
        cur = nxt;
    }
}

template <int CP, int R, bool ALIGNED>
__global__ void __launch_bounds__(128, 4)
k_walk4e(const WalkArgs A) {
    walk4eBody<double, CP, R, ALIGNED>(A);
}

// fp32 partials storage (PRECISION_SINGLE)
template <int CP, int R, bool ALIGNED>
__global__ void __launch_bounds__(128, 4)
k_walk4es(const WalkArgs A) {
    walk4eBody<float, CP, R, ALIGNED>(A);
}

// ---------------------------------------------------------------------------------------------------------------------
// k_walk4p -- the same arithmetic with PER-WARP ASYNCHRONOUS OPERAND STAGING (every aligned list at CP <= 8).
//
// What bounds k_walk4e with the matrices gone: no pipe near its peak, but "long scoreboard" stalls on first uses of
// small per-op operands -- the op record, the tips' state bytes, the
// spectra, the P columns of tip children -- i.e. a chain of dependent L1/L2 latencies per op with 16 warps per SM to hide it.
// Those operands are tiny, warp-uniform and known one op ahead, so each warp runs a two-deep cp.async (LDGSTS) pipeline into
// its own slice of shared memory: while op k computes, record k+2 and ALL small operands of op k+1 travel global -> shared
// without touching a register; op k+1 finds them with shared-memory latency.  Per op and warp: three LDGSTS instructions.
//   ring[4]            op records (64 B), fetched two ops ahead (k_walk4pv: with the tips of their virtual children)
//   stage[k & 1]       mat[child][2][5*CP][2] P block of a tip child: the contiguous [j][CP][i] block in HBM travels as 16-byte
//                                            pieces, one per lane, and every piece lands where the READS are conflict-free:
//                                            two half tables (states 0-1 / 2-3) of 16-byte entries indexed c*4 + j, so that
//                                            the 8 lanes of a quarter warp (same category, 8 patterns) hit 4 distinct
//                                            bank groups whatever their states -- with the HBM order kept ([j][c]: 128 B
//                                            between states) they collided up to 4-way and most of the kernel's shared-memory
//                                            wavefronts were bank conflicts.  Entries
//                                            4*CP + c = the gap column (written once).  A pattern picks its column with two LDS.128
//                      ev[child][CP][4]      spectrum of an internal child
//                      st[child][G*R]        state bytes of a tip child for this warp's patterns
// Child partials that are not forwarded in registers keep the look-ahead L1 prefetch.  Aligned lists only (every op spans
// [0, Ppad)), thin R = 1 phases included; pattern windows (by-partition lists) use k_walk4e.
//
// VIRTUAL CHERRIES (k_walk4pv): a cherry (tip x tip op, no rescaling) is a pure function of two state bytes per pattern and
// two P blocks, so api.cu does not run it at all: its consumers recompute it where they read it.  A virtual child (Op4 flag
// bit 2 / 3) names the cherry's buffer, whose recipe row holds the two P blocks ([2][j][CP][i], copied by k_cherry_snapshot
// when the cherry was produced); its two tips travel in a parallel per-op array (one more lane of the record fetch).  Its staging is that of two tip children (tables
// mat[ch] / mat[2 + ch], state bytes st[ch] / st[2 + ch]) plus the spectrum of the consumer's branch; its value
// x = colA ⊙ colB is the very product the cherry op would have stored, so everything downstream is bit-identical.
//
// SIBLING STACK: a result that a later op of the same walk reads, but not from registers (the sibling of some later op),
// is also kept in a per-warp slot of dynamic shared memory (Op4 slot bytes, assigned by api.cu::assignStackSlots), and
// that later op reads the slot instead of global memory.  Layout [slot][warp][R][2][32] 16-byte entries: lane fastest,
// so every STS.128 / LDS.128 is conflict-free.  A thread reads back only cells it wrote itself: program order suffices.
// The slot holds the rounded cell that was stored, so the value does not depend on the route it takes.
__device__ __forceinline__ void cpAsync16(void* smemDst, const void* gmemSrc) {
    const unsigned sAddr = (unsigned)__cvta_generic_to_shared(smemDst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"(sAddr), "l"(gmemSrc) : "memory");
}
template <int BYTES>
__device__ __forceinline__ void cpAsyncSmall(void* smemDst, const void* gmemSrc) {      // 4, 8 or 16 bytes
    const unsigned sAddr = (unsigned)__cvta_generic_to_shared(smemDst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" :: "r"(sAddr), "l"(gmemSrc), "n"(BYTES) : "memory");
}

// one cell of the sibling stack: two 16-byte entries 32 entries (one per lane) apart.  volatile, like the global cell
// accesses, so that ptxas schedules a slot read where the load it replaces would have been
__device__ __forceinline__ void lds256(const double2* p, double (&v)[4]) {
    const unsigned a = (unsigned)__cvta_generic_to_shared(p);
    asm volatile("ld.shared.v2.f64 {%0,%1}, [%4];\n\tld.shared.v2.f64 {%2,%3}, [%4+512];"
                 : "=d"(v[0]), "=d"(v[1]), "=d"(v[2]), "=d"(v[3]) : "r"(a) : "memory");
}
__device__ __forceinline__ void sts256(double2* p, const double (&v)[4]) {
    const unsigned a = (unsigned)__cvta_generic_to_shared(p);
    asm volatile("st.shared.v2.f64 [%0], {%1,%2};\n\tst.shared.v2.f64 [%0+512], {%3,%4};"
                 :: "r"(a), "d"(v[0]), "d"(v[1]), "d"(v[2]), "d"(v[3]) : "memory");
}

// dynamic shared memory of a 4-warp block's sibling stack: [slot][warp][R][2][32] 16-byte entries
constexpr size_t stackBytes(int slots, int R) { return (size_t)slots * 4 * R * 64 * sizeof(double2); }
// the instances that carry the sibling stack: CP = 4, launched at 3 blocks per SM.  ptxas keeps them without a spill and
// the stack keeps their 3 blocks per SM; at other category counts the slot code would cost spills or blocks, so those
// instances are built without it and ignore the slot bytes
__host__ __device__ constexpr bool stackBuilt(int CP) { return CP == 4; }
// launch bound of k_walk4p / k_walk4ps: 3 blocks let ptxas keep CP = 4 without a spill and 4 blocks still fit -- the
// fastest setting where it was swept (BASELINE.md 6.7)
constexpr int stagedMinBlocks(int CP) { return CP == 4 ? 3 : 4; }

template <int CP, int R, bool VIRT>
struct WarpStage {
    static constexpr int G = 32 / CP, NP = G * R, TABLES = VIRT ? 4 : 2;
    double mat[TABLES][5 * CP * 4];
    double ev[2][CP * 4];
    alignas(16) unsigned char st[TABLES][NP < 16 ? 16 : NP];
};

template <typename T, int CP, int R, bool VIRT, bool STACK>
__device__ __forceinline__ void walk4pBody(const WalkArgs& A) {
    constexpr int G = 32 / CP, NP = G * R;
    constexpr int PIECE = NP < 16 ? NP : 16;                       // state bytes travel in 4-, 8- or 16-byte pieces
    static_assert(NP % PIECE == 0 && (PIECE == 4 || PIECE == 8 || PIECE == 16), "state-byte staging");
    constexpr int TABLES = WarpStage<CP, R, VIRT>::TABLES;
    constexpr int RECQ = sizeof(Op4) / 16 + (VIRT ? 1 : 0);        // 16-byte pieces of one op record (+ its virtual tips)
    __shared__ __align__(16) WarpStage<CP, R, VIRT> stages[4][2];
    __shared__ __align__(16) Op4 rings[4][4];
    __shared__ __align__(16) int4 tipRings[4][VIRT ? 4 : 1];
    extern __shared__ double2 sibStack[];
    int lane;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));            // volatile: never rematerialised as an S2R inside the loop
    const int wib = threadIdx.x >> 5;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int c = lane / G;
    const int4 range = __ldg(A.subs + blockIdx.y);
    const int pBase = range.z + warp * NP;                         // first pattern of this warp
    if (pBase >= range.w) return;
    const int p0 = pBase + (lane % G);                             // patterns p0 + r*G
    const bool catValid = c < A.C;
    const int cc = catValid ? c : 0;
    const size_t off0 = ((size_t)cc * A.Ppad + p0) * 4;
    const int last = range.y - 1, S = A.S;
    WarpStage<CP, R, VIRT>* stage = stages[wib];
    Op4* ring = rings[wib];
    int4* tipRing = tipRings[wib];
    double2* const myStack = sibStack + wib * R * 64 + lane;       // + (slot * 4 * R + r) * 64, halves 32 entries apart

    // the gap column (row 4 of every table), once
    for (int q = lane; q < 2 * TABLES * CP * 4; q += 32) {
        const int tbl = q / (CP * 4), e = q % (CP * 4), gc = e >> 2, i = e & 3;
        stage[tbl / TABLES].mat[tbl % TABLES][(i >> 1) * 10 * CP + 2 * (4 * CP + gc) + (i & 1)] = (i < S) ? 1.0 : 0.0;
    }
    // P block [j][CP][i] (4 * CP * 4 doubles, contiguous) -> table: piece q = (j, c, half) -> half table, entry c*4 + j
    auto stageBlock = [&](double* tab, const double* src) {
#pragma unroll
        for (int q = lane; q < CP * 8; q += 32)
            cpAsync16(&tab[(q & 1) * 10 * CP + 2 * (((q >> 1) % CP) * 4 + q / (2 * CP))], src + 2 * q);
    };
    // lanes 0 .. RECQ-1: record j into the ring (k_walk4pv: lane 4 brings the tips of its virtual children)
    auto fetchRecord = [&](int j) {
        if (VIRT && lane == RECQ - 1) cpAsync16(&tipRing[j & 3], A.virtTips + j);
        else cpAsync16(reinterpret_cast<char*>(&ring[j & 3]) + 16 * lane, reinterpret_cast<const char*>(A.ops + j) + 16 * lane);
    };
    // what op j reads beyond partials goes to stage j & 1; reads record j from the ring (it has arrived) ONCE -- the fields
    // the compute part needs travel on in registers (4 shared-memory reads per op instead of 20)
    struct Rec { int dest, c1, c2, sw, sr, flags, pfA, pfB, slots; };
    auto issueOperands = [&](int j) -> Rec {
        const int4 rec = *reinterpret_cast<const int4*>(&ring[j & 3]);          // dest, c1, c2, m1
        const int4 rec2 = *(reinterpret_cast<const int4*>(&ring[j & 3]) + 1);   // m2, sw, sr, cum
        const int flags = ring[j & 3].pad_;
        const int slots = STACK ? (int)ring[j & 3].slots : 0xFFFFFF;
        const int2 pf = *reinterpret_cast<const int2*>(&ring[j & 3].pfA);
        const int m2 = rec2.x;
        WarpStage<CP, R, VIRT>& sg = stage[j & 1];
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
            const int child = ch == 0 ? rec.y : rec.z, m = ch == 0 ? rec.w : m2;
            const bool virt = VIRT && (flags & (4 << ch)) != 0;
            if (child < 0) {
                stageBlock(sg.mat[ch], A.mats + (size_t)m * A.matStride);
            } else {
                if (virt) {
                    const double* rcp = A.recipes + (size_t)child * 32 * CP;
                    stageBlock(sg.mat[ch], rcp);
                    stageBlock(sg.mat[TABLES - 2 + ch], rcp + 16 * CP);
                }
                if (lane < CP * 2) cpAsync16(&sg.ev[ch][2 * lane], A.evecs + (size_t)m * CP * 4 + 2 * lane);
            }
        }
        // one more instruction: record j + 1 on lanes 0 .. RECQ-1, then the state bytes of the tip children and of the
        // virtual children's tips (set t = table t)
        constexpr int SL = NP / PIECE;
        auto statePiece = [&](int q) {                             // piece q of all state-byte sets
            const int t = q / SL, piece = q % SL, ch = t & 1;
            const int child = ch == 0 ? rec.y : rec.z;
            int tip = t < 2 && child < 0 ? -child - 1 : -1;
            if (VIRT && (flags & (4 << ch)) != 0) {
                const int4 vt = tipRing[j & 3];                      // tips of virtual child 1 (x, y), 2 (z, w)
                tip = t == 0 ? vt.x : t == 1 ? vt.z : t == 2 ? vt.y : vt.w;
            }
            if (tip >= 0) cpAsyncSmall<PIECE>(&sg.st[t][PIECE * piece], A.states + (size_t)tip * A.Ppad + pBase + PIECE * piece);
        };
        if (lane < RECQ) {
            if (j + 1 <= last) fetchRecord(j + 1);
        } else if (lane < RECQ + TABLES * SL) {
            statePiece(lane - RECQ);
        }
        if constexpr (RECQ + TABLES * SL > 32) {
            if (lane < RECQ + TABLES * SL - 32) statePiece(lane + 32 - RECQ);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        return Rec{rec.x, rec.y, rec.z, rec2.y, rec2.z, flags, pf.x, pf.y, slots};
    };
    // prologue: records k0 (and k0+1 through issueOperands), then the operands of k0
    if (lane < RECQ) fetchRecord(range.x);
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    Rec nxt = issueOperands(range.x);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();

    double Vi[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) asm volatile("mov.f64 %0, %1;" : "=d"(Vi[q]) : "d"(A.Vi[q]));
    double d[R][4];
#pragma unroll
    for (int r = 0; r < R; ++r) d[r][0] = d[r][1] = d[r][2] = d[r][3] = 0.0;

    for (int k = range.x; k <= last; ++k) {
        const Rec cur = nxt;
        if (k + 1 <= last) nxt = issueOperands(k + 1);             // travels while op k computes
        const WarpStage<CP, R, VIRT>& sg = stage[k & 1];
        // look-ahead for the child partials of op k+1 that are not forwarded (never this op's destination)
#pragma unroll
        for (int w = 0; w < 2; ++w) {
            const int pf = w == 0 ? cur.pfA : cur.pfB;
            if (pf == 0 || (pf & 1) || !catValid) continue;
            const T* xg = static_cast<const T*>(A.partials) + (size_t)((pf >> 1) - 1) * A.stride + off0;
#pragma unroll
            for (int r = 0; r < R; ++r) prefetchL1(xg + (size_t)r * G * 4);
        }
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
            const int child = ch == 0 ? cur.c1 : cur.c2;
            if (child < 0) {
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const int sym = sg.st[ch][(lane % G) + r * G];
                    const int e2 = 2 * (sym < S ? cc * 4 + sym : 4 * CP + cc);
                    const double2 lo = *reinterpret_cast<const double2*>(&sg.mat[ch][e2]);
                    const double2 hi = *reinterpret_cast<const double2*>(&sg.mat[ch][10 * CP + e2]);
                    if (ch == 0) { d[r][0] = lo.x; d[r][1] = lo.y; d[r][2] = hi.x; d[r][3] = hi.y; }
                    else { d[r][0] *= lo.x; d[r][1] *= lo.y; d[r][2] *= hi.x; d[r][3] *= hi.y; }
                }
            } else {
                const double2* ep = reinterpret_cast<const double2*>(&sg.ev[ch][cc * 4]);
                const double2 e01 = ep[0], e23 = ep[1];
                const double e[4] = {e01.x, e01.y, e23.x, e23.y};
                const bool fromRegisters = ch == 0 && (cur.flags & 2) != 0;
                const bool virt = VIRT && (cur.flags & (4 << ch)) != 0;
                const int src = STACK ? (cur.slots >> (8 * ch)) & 0xFF : 0xFF;
                const T* xg = static_cast<const T*>(A.partials) + (size_t)child * A.stride + off0;
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    double x[4], u[4], y[4];
                    if (fromRegisters) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) x[i] = d[r][i];
                    } else if (virt) {                                  // the cherry's value, as its op would have stored it
                        const int symA = sg.st[ch][(lane % G) + r * G], symB = sg.st[TABLES - 2 + ch][(lane % G) + r * G];
                        const int eA = 2 * (symA < S ? cc * 4 + symA : 4 * CP + cc);
                        const int eB = 2 * (symB < S ? cc * 4 + symB : 4 * CP + cc);
                        const double2 aLo = *reinterpret_cast<const double2*>(&sg.mat[ch][eA]);
                        const double2 aHi = *reinterpret_cast<const double2*>(&sg.mat[ch][10 * CP + eA]);
                        const double2 bLo = *reinterpret_cast<const double2*>(&sg.mat[TABLES - 2 + ch][eB]);
                        const double2 bHi = *reinterpret_cast<const double2*>(&sg.mat[TABLES - 2 + ch][10 * CP + eB]);
                        x[0] = aLo.x * bLo.x; x[1] = aLo.y * bLo.y; x[2] = aHi.x * bHi.x; x[3] = aHi.y * bHi.y;
                        roundCell<T>(x);
                    } else if (STACK && src != 0xFF) {                  // a sibling this thread parked earlier
                        lds256(myStack + (src * 4 * R + r) * 64, x);
                    } else {
                        loadCell(xg + (size_t)r * G * 4, x);
                    }
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        u[q] = (Vi[4 * q] * x[0] + Vi[4 * q + 1] * x[1] + Vi[4 * q + 2] * x[2] + Vi[4 * q + 3] * x[3]) * e[q];
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        y[i] = absBits(A.V[4 * i] * u[0] + A.V[4 * i + 1] * u[1] + A.V[4 * i + 2] * u[2] + A.V[4 * i + 3] * u[3]);
#pragma unroll
                    for (int i = 0; i < 4; ++i) d[r][i] = ch == 0 ? y[i] : d[r][i] * y[i];
                }
            }
        }
        T* dg = static_cast<T*>(A.partials) + (size_t)cur.dest * A.stride + off0;
        const int dst = STACK ? (cur.slots >> 16) & 0xFF : 0xFF;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int p = p0 + r * G;
            if (cur.sw >= 0) {                 // rescaling (AbstractLikelihoodCore.java:406-442, unconditional as in BEAGLE)
                double m = catValid ? fmax(fmax(d[r][0], d[r][1]), fmax(d[r][2], d[r][3])) : 0.0;
#pragma unroll
                for (int sh = G; sh < 32; sh <<= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, sh));
                if (m == 0.0) m = 1.0;
                const double inv = 1.0 / m;
#pragma unroll
                for (int i = 0; i < 4; ++i) d[r][i] *= inv;
                if (c == 0) A.scale[(size_t)cur.sw * A.Ppad + p] = A.logScalers ? log(m) : m;
            } else if (cur.sr >= 0) {
                double f = A.scale[(size_t)cur.sr * A.Ppad + p];
                if (A.logScalers) f = exp(f);
                const double inv = 1.0 / f;
#pragma unroll
                for (int i = 0; i < 4; ++i) d[r][i] *= inv;
            }
            roundCell<T>(d[r]);
            if (catValid) storeCell(dg + (size_t)r * G * 4, d[r]);
            if (STACK && dst != 0xFF) sts256(myStack + (dst * 4 * R + r) * 64, d[r]);
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");      // op k+1's operands and record k+2 have landed
        __syncwarp();
    }
}

template <int CP, int R>
__global__ void __launch_bounds__(128, stagedMinBlocks(CP))
k_walk4p(const WalkArgs A) {
    walk4pBody<double, CP, R, false, stackBuilt(CP)>(A);
}

template <int CP, int R>
__global__ void __launch_bounds__(128, stagedMinBlocks(CP))
k_walk4ps(const WalkArgs A) {
    walk4pBody<float, CP, R, false, stackBuilt(CP)>(A);
}

// lists that read virtual cherries: twice the tip tables per warp stage.  One launch bound: with 3 blocks ptxas keeps the
// doubled staging of k_walk4pv in registers without a spill at every CP and R
template <int CP, int R>
__global__ void __launch_bounds__(128, 3)
k_walk4pv(const WalkArgs A) {
    walk4pBody<double, CP, R, true, stackBuilt(CP)>(A);
}

template <int CP, int R>
__global__ void __launch_bounds__(128, 3)
k_walk4pvs(const WalkArgs A) {
    walk4pBody<float, CP, R, true, stackBuilt(CP)>(A);
}

// stackSlots: the sibling stack of the phase (dynamic shared memory; 0 on instances built without it).  The kernel's
// limit is set once per device to the deepest stack it can get (kStackSlots slots), never lowered: instances on other host
// threads launch the same kernel with other depths.  No carveout preference: the driver sizes shared memory per launch, so
// launches without a stack keep the larger L1.
template <auto KERNEL, int CP, int R>
cudaError_t launchStaged(Instance* in, const WalkArgs& A, dim3 grid, int stackSlots) {
    const size_t smem = stackBuilt(CP) ? stackBytes(stackSlots, R) : 0;
    if (smem > 0) {
        static std::atomic<unsigned long long> limitSet{0};             // one bit per device
        const unsigned long long bit = 1ull << (in->device & 63);
        if (!(limitSet.load() & bit)) {
            cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 (int)stackBytes(kStackSlots, R));
            if (e != cudaSuccess) return e;
            limitSet.fetch_or(bit);
        }
    }
    if (in->debugLog) {
        const auto kernel = KERNEL;
        int blocks = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kernel, 128, smem);
        fprintf(stderr, "[b200-beagle] staged walk: %zu B sibling stack per block, %d blocks per SM\n", smem, blocks);
    }
    KERNEL<<<grid, 128, smem, in->stream>>>(A);
    return cudaGetLastError();
}

// the kernel of one (CP, R) for the route's family and the instance's precision: the staged kernels and fp32 storage are
// built for CP <= 8, the ALIGNED k_walk4e for CP 16 and 32
template <int CP, int R>
cudaError_t launchEigenWalk(Instance* in, Walk4Kernel kernel, const WalkArgs& A, dim3 grid, int stackSlots) {
    const bool s = in->single;
    if constexpr (CP <= 8) {
        switch (kernel) {
            case Walk4Kernel::Staged:
                return s ? launchStaged<k_walk4ps<CP, R>, CP, R>(in, A, grid, stackSlots)
                         : launchStaged<k_walk4p<CP, R>, CP, R>(in, A, grid, stackSlots);
            case Walk4Kernel::StagedVirtual:
                return s ? launchStaged<k_walk4pvs<CP, R>, CP, R>(in, A, grid, stackSlots)
                         : launchStaged<k_walk4pv<CP, R>, CP, R>(in, A, grid, stackSlots);
            case Walk4Kernel::EigenPredicated:
                if (s) k_walk4es<CP, R, false><<<grid, 128, 0, in->stream>>>(A);
                else k_walk4e<CP, R, false><<<grid, 128, 0, in->stream>>>(A);
                return cudaGetLastError();
            default: return cudaErrorInvalidValue;
        }
    } else {
        if (s) return cudaErrorInvalidValue;
        switch (kernel) {
            case Walk4Kernel::EigenAligned: k_walk4e<CP, R, true><<<grid, 128, 0, in->stream>>>(A); return cudaGetLastError();
            case Walk4Kernel::EigenPredicated: k_walk4e<CP, R, false><<<grid, 128, 0, in->stream>>>(A); return cudaGetLastError();
            default: return cudaErrorInvalidValue;
        }
    }
}

// recipe rows [buffer][2][16 * CP] of the virtual cherries a list produces: items (buffer, m1, m2, -)
__global__ void k_cherry_snapshot(const int4* items, const double* mats, size_t matStride, double* recipes, int blk) {
    const int4 it = items[blockIdx.x];
    for (int q = threadIdx.x; q < 2 * blk; q += blockDim.x)
        recipes[(size_t)it.x * 2 * blk + q] = mats[(size_t)(q < blk ? it.y : it.z) * matStride + q % blk];
}

// stored partials of virtual cherries, from their recipes: items (slot, buffer, tip 1, tip 2), grid.y strides over them;
// the same lookups and the same product as k_walk4p's tip tables, so the stored value is the one the cherry op would have
// written
template <typename T>
__device__ __forceinline__ void cherryStoreBody(const int4* items, int count, T* partials, size_t stride,
                                                const uint8_t* states, const double* recipes, int S, int C, int CP, int Ppad) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= C * Ppad) return;
    const int c = q / Ppad, p = q - c * Ppad;
    for (int k = blockIdx.y; k < count; k += gridDim.y) {
        const int4 it = items[k];
        const int sA = states[(size_t)it.z * Ppad + p], sB = states[(size_t)it.w * Ppad + p];
        const double* ra = recipes + (size_t)it.y * 32 * CP;
        const double* rb = ra + 16 * CP;
        double v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const double a = sA < S ? ra[(sA * CP + c) * 4 + i] : (i < S ? 1.0 : 0.0);
            const double b = sB < S ? rb[(sB * CP + c) * 4 + i] : (i < S ? 1.0 : 0.0);
            v[i] = a * b;
        }
        roundCell<T>(v);
        storeCell(partials + (size_t)it.x * stride + (size_t)q * 4, v);
    }
}

__global__ void k_cherry_store(const int4* items, int count, double* partials, size_t stride, const uint8_t* states,
                               const double* recipes, int S, int C, int CP, int Ppad) {
    cherryStoreBody(items, count, partials, stride, states, recipes, S, C, CP, Ppad);
}

__global__ void k_cherry_store_f32(const int4* items, int count, float* partials, size_t stride, const uint8_t* states,
                                const double* recipes, int S, int C, int CP, int Ppad) {
    cherryStoreBody(items, count, partials, stride, states, recipes, S, C, CP, Ppad);
}

}  // namespace

bool walkStackBuilt(const Instance* in) { return stackBuilt(in->matCP); }

Walk4Route walk4Route(const Instance* in, int nSubs, int maxWindow, bool eigenForm, bool aligned, bool virt) {
    const int CP = in->matCP, G = 32 / CP;
    // a thin phase (few walks in flight) is latency-bound: one pattern group per thread gives the most warps per op
    const long walks = (long)nSubs * ((maxWindow + G * in->walkR - 1) / (G * in->walkR));
    Walk4Route r{Walk4Kernel::Unservable, in->walkR, walks < (long)in->smCount * 8};
    if (in->thinR1 && r.thin) r.R = 1;
    else if (eigenForm && r.R > 1) r.R = CP == 4 && in->walkR == 2 ? 2 : 4;     // the eigen form builds R = 2 at CP = 4 only
    if (in->single && CP > 8) return r;                  // fp32 storage is built for CP <= 8 (single instances have C <= 8)
    if (!eigenForm) {
        if (!virt) r.kernel = Walk4Kernel::Matrix;       // only the staged eigen-form kernels read virtual cherries
        return r;
    }
    // predicate-free only when a warp's G * R patterns can never straddle the end of the padded pattern axis; the staged
    // kernels need at least 4 patterns per warp
    const bool whole = aligned && in->Ppad % (G * r.R) == 0;
    if (whole && CP <= 8 && G * r.R >= 4) r.kernel = virt ? Walk4Kernel::StagedVirtual : Walk4Kernel::Staged;
    else if (!virt) r.kernel = whole && CP > 8 ? Walk4Kernel::EigenAligned : Walk4Kernel::EigenPredicated;
    return r;
}

// eigen: [V (16, row-major Evec[i][k]) | V^-1 (16, Ievc[k][j])], padded to 4 x 4 with zeros
cudaError_t launchWalk4E(Instance* in, const Walk4Route& route, const Op4* dOps, const int4* dSubs, int nSubs, int maxWindow,
                         const double* eigen, const int4* dVirtTips, int stackSlots) {
    if (route.kernel == Walk4Kernel::StagedVirtual && in->dRecipe == nullptr) return cudaErrorInvalidValue;
    WalkArgs A = walkArgs(in, dOps, dSubs);
    A.evecs = in->dEvec;
    A.recipes = in->dRecipe;
    A.virtTips = dVirtTips;
    for (int q = 0; q < 16; ++q) { A.V[q] = eigen[q]; A.Vi[q] = eigen[16 + q]; }
    const dim3 grid = walkGrid(in->matCP, route.R, nSubs, maxWindow);
    switch (in->matCP * 8 + route.R) {                             // (CP, R)
        case 1 * 8 + 1: return launchEigenWalk<1, 1>(in, route.kernel, A, grid, stackSlots);
        case 1 * 8 + 4: return launchEigenWalk<1, 4>(in, route.kernel, A, grid, stackSlots);
        case 2 * 8 + 1: return launchEigenWalk<2, 1>(in, route.kernel, A, grid, stackSlots);
        case 2 * 8 + 4: return launchEigenWalk<2, 4>(in, route.kernel, A, grid, stackSlots);
        case 4 * 8 + 1: return launchEigenWalk<4, 1>(in, route.kernel, A, grid, stackSlots);
        case 4 * 8 + 2: return launchEigenWalk<4, 2>(in, route.kernel, A, grid, stackSlots);
        case 4 * 8 + 4: return launchEigenWalk<4, 4>(in, route.kernel, A, grid, stackSlots);
        case 8 * 8 + 1: return launchEigenWalk<8, 1>(in, route.kernel, A, grid, stackSlots);
        case 8 * 8 + 4: return launchEigenWalk<8, 4>(in, route.kernel, A, grid, stackSlots);
        case 16 * 8 + 1: return launchEigenWalk<16, 1>(in, route.kernel, A, grid, stackSlots);
        case 16 * 8 + 4: return launchEigenWalk<16, 4>(in, route.kernel, A, grid, stackSlots);
        case 32 * 8 + 1: return launchEigenWalk<32, 1>(in, route.kernel, A, grid, stackSlots);
        case 32 * 8 + 4: return launchEigenWalk<32, 4>(in, route.kernel, A, grid, stackSlots);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launchCherrySnapshot(Instance* in, const int4* dItems, int count) {
    if (count <= 0) return cudaSuccess;
    k_cherry_snapshot<<<count, 128, 0, in->stream>>>(dItems, in->dMat, in->matStride, in->dRecipe, 16 * in->matCP);
    return cudaGetLastError();
}

cudaError_t launchCherryStore(Instance* in, const int4* dItems, int count) {
    if (count <= 0) return cudaSuccess;
    const dim3 grid((in->C * in->Ppad + 255) / 256, std::min(count, 65535));
    if (in->single)
        k_cherry_store_f32<<<grid, 256, 0, in->stream>>>(dItems, count, reinterpret_cast<float*>(in->partialsBase),
                                                      in->partialsElems, in->states8Base, in->dRecipe, in->S, in->C,
                                                      in->matCP, in->Ppad);
    else
        k_cherry_store<<<grid, 256, 0, in->stream>>>(dItems, count, reinterpret_cast<double*>(in->partialsBase),
                                                     in->partialsElems, in->states8Base, in->dRecipe, in->S, in->C,
                                                     in->matCP, in->Ppad);
    return cudaGetLastError();
}

cudaError_t updateWalk4EGraph(cudaGraphExec_t exec, const std::vector<cudaGraphNode_t>& kernelNodes, const double* eigen) {
    for (cudaGraphNode_t node : kernelNodes) {
        cudaKernelNodeParams kp;
        cudaError_t e = cudaGraphKernelNodeGetParams(node, &kp);
        if (e != cudaSuccess) return e;
        if (kp.func == reinterpret_cast<void*>(k_cherry_snapshot)) continue;     // carries no eigen system
        if (kp.kernelParams == nullptr || kp.kernelParams[0] == nullptr) return cudaErrorInvalidValue;
        WalkArgs A = *static_cast<const WalkArgs*>(kp.kernelParams[0]);       // every eigen-form walk kernel takes ONE WalkArgs
        for (int q = 0; q < 16; ++q) { A.V[q] = eigen[q]; A.Vi[q] = eigen[16 + q]; }
        void* args[1] = {&A};
        kp.kernelParams = args;
        kp.extra = nullptr;
        e = cudaGraphExecKernelNodeSetParams(exec, node, &kp);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace b200
