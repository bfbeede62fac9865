// walk4.cuh -- device helpers and launch arguments shared by the 4-state walk kernels (kernels.cu, walk4e.cu).
#pragma once
#include "engine.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// small device helpers
// ---------------------------------------------------------------------------------------------
// 32 contiguous bytes (one pattern's 4 states) as two 128-bit accesses: sm_90 has no 256-bit global load/store
__device__ __forceinline__ void ldg256(const double* p, double (&v)[4]) {
    asm volatile("ld.global.v2.f64 {%0,%1}, [%4];\n\tld.global.v2.f64 {%2,%3}, [%4+16];"
                 : "=d"(v[0]), "=d"(v[1]), "=d"(v[2]), "=d"(v[3]) : "l"(p) : "memory");
}
// read-only path for data produced by an EARLIER launch (matrices)
__device__ __forceinline__ void ldg256_nc(const double* p, double (&v)[4]) {
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%4];\n\tld.global.nc.v2.f64 {%2,%3}, [%4+16];"
                 : "=d"(v[0]), "=d"(v[1]), "=d"(v[2]), "=d"(v[3]) : "l"(p));
}
__device__ __forceinline__ void stg256(double* p, const double (&v)[4]) {
    asm volatile("st.global.v2.f64 [%0], {%1,%2};\n\tst.global.v2.f64 [%0+16], {%3,%4};"
                 :: "l"(p), "d"(v[0]), "d"(v[1]), "d"(v[2]), "d"(v[3]) : "memory");
}

// ---- the partials cell of one pattern (4 states): the one place on the device that knows the storage format.
// T = double: 32 bytes as two 128-bit accesses.  T = float (PRECISION_SINGLE instances): 16 bytes as one 128-bit access,
// widened to double on load.  Arithmetic is fp64 either way.  A float instance rounds every partials value before anyone
// reads it -- stored, forwarded in registers or recomputed (roundCell) -- so the route a value takes never shows.
// The rounding is that of cvt.rn.ftz.f32.f64: round to nearest, a subnormal result becomes a zero of the same sign (done
// here on the integer pipe: ptxas emulates the .ftz of that cvt with an FP64 compare, and the FP64 pipe is the busy one).
template <typename T>
__device__ __forceinline__ void roundCell(double (&v)[4]) {
    if constexpr (sizeof(T) == 4) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float f;
            asm("cvt.rn.f32.f64 %0, %1;" : "=f"(f) : "d"(v[i]));
            const unsigned b = __float_as_uint(f);
            v[i] = (double)((b & 0x7f800000u) ? f : __uint_as_float(b & 0x80000000u));
        }
    }
}
__device__ __forceinline__ void loadCell(const double* p, double (&v)[4]) { ldg256(p, v); }
__device__ __forceinline__ void loadCell(const float* p, double (&v)[4]) {
    float f[4];
    asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(f[0]), "=f"(f[1]), "=f"(f[2]), "=f"(f[3]) : "l"(p) : "memory");
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = f[i];
}
// v must have been through roundCell<T>: the narrowing below is then exact
__device__ __forceinline__ void storeCell(double* p, const double (&v)[4]) { stg256(p, v); }
__device__ __forceinline__ void storeCell(float* p, const double (&v)[4]) {
    asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"((float)v[0]), "f"((float)v[1]), "f"((float)v[2]), "f"((float)v[3]) : "memory");
}

struct WalkArgs {
    const Op4* ops;
    const int4* subs;          // [subtree] = (first op, one-past-last op, first pattern, one-past-last pattern)
    void* partials;            // slab base: double, or float on a PRECISION_SINGLE instance (stride counts elements)
    size_t stride;             // elements per slot
    const uint8_t* states;     // [tip][Ppad]
    const double* mats;        // [matrix][4][CP][4]
    double* scale;             // [buffer][Ppad]
    int S, C, Ppad, logScalers;
    size_t matStride;          // elements per matrix buffer
    // eigen-form walk (walk4e.cu): per-branch spectra exp(lambda_k r_c t) [matrix][CP][4] in HBM, and the ONE eigen system
    // of the list by value -- kernel parameters live in the constant bank, so V / V^-1 cost neither registers nor LSU
    // traffic (DFMA takes them as uniform-register operands)
    const double* evecs;
    const double* recipes;     // virtual cherries: [buffer][2][16 * CP], the two P blocks each was computed with
    const int4* virtTips;      // [op] the tips of its virtual children (child 1: x, y; child 2: z, w)
    double V[16];              // Evec[i][k], rows/columns >= S zero
    double Vi[16];             // Ievc[k][j]
};

// the fields both forms fill from the instance (the eigen form adds its own)
inline WalkArgs walkArgs(const Instance* in, const Op4* dOps, const int4* dSubs) {
    WalkArgs A;
    A.ops = dOps; A.subs = dSubs; A.partials = in->partialsBase; A.stride = in->partialsElems;
    A.states = in->states8Base; A.mats = in->dMat; A.scale = in->dScale;
    A.S = in->S; A.C = in->C; A.Ppad = in->Ppad; A.logScalers = in->logScalers ? 1 : 0;
    A.matStride = in->matStride;
    return A;
}

// 128-thread blocks of 4 warps, a warp per 32 / CP * R patterns of the window; one grid row per subtree walk
inline dim3 walkGrid(int CP, int R, int nSubs, int maxWindow) {
    const int G = 32 / CP, warps = (maxWindow + G * R - 1) / (G * R);
    return dim3((warps + 3) / 4, nSubs);
}

__device__ __forceinline__ Op4 loadOp(const Op4* p) {
    const int4* q = reinterpret_cast<const int4*>(p);
    int4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
    Op4 o;
    o.dest = a.x; o.c1 = a.y; o.c2 = a.z; o.m1 = a.w;
    o.m2 = b.x; o.sw = b.y; o.sr = b.z; o.cum = b.w;
    o.pBegin = c.x; o.pEnd = c.y; o.slots = (unsigned)c.z; o.pad_ = c.w;
    o.pfA = d.x; o.pfB = d.y; o.pfM1 = d.z; o.pfM2 = d.w;
    return o;
}

__device__ __forceinline__ void prefetchL1(const void* p) {
    asm volatile("prefetch.global.L1 [%0];" :: "l"(p));
}

// non-volatile: a read-only load the scheduler may hoist freely
__device__ __forceinline__ void ldg256_ro(const double* p, double (&v)[4]) {
    asm("ld.global.nc.v2.f64 {%0,%1}, [%4];\n\tld.global.nc.v2.f64 {%2,%3}, [%4+16];"
        : "=d"(v[0]), "=d"(v[1]), "=d"(v[2]), "=d"(v[3]) : "l"(p));
}
// a partials cell an EARLIER launch wrote, on the same non-volatile read-only path
__device__ __forceinline__ void loadCellRo(const double* p, double (&v)[4]) { ldg256_ro(p, v); }
__device__ __forceinline__ void loadCellRo(const float* p, double (&v)[4]) {
    float f[4];
    asm("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(f[0]), "=f"(f[1]), "=f"(f[2]), "=f"(f[3]) : "l"(p));
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = f[i];
}

}  // namespace b200
