/*
 * ORACLE -- test infrastructure only (checker and cpu_baseline; never linked into the product).
 *
 * Plain C (fp64, pthreads) restatement of the four BEAGLE calls on BEAST's tree-likelihood hot
 * path, i.e. a "BEAGLE-CPU-equivalent restatement" (BASELINE.md section 4): the reference's real CPU
 * path is the un-vendored beagle-lib, which cannot be built here.  The arithmetic follows the
 * reference's in-tree statements of the same algorithm:
 *   pruning ...................... src/dr/oldevomodel/treelikelihood/GeneralLikelihoodCore.java:52-203
 *   category integration, root ... GeneralLikelihoodCore.java:358-408
 *   rescaling / accumulation ..... src/dr/oldevomodel/treelikelihood/AbstractLikelihoodCore.java:406-459
 *   P(t) from the eigen system ... src/dr/evomodel/substmodel/BaseSubstitutionModel.java:206-241
 *   op tuples .................... src/dr/evomodel/treedatalikelihood/BeagleDataLikelihoodDelegate.java:857-937
 * Threads split the patterns into contiguous blocks (what BEAGLE-CPU's setCPUThreadCount does,
 * BDLD:482-499); every block walks the whole op list, which is legal because pattern columns are
 * independent.  Pinned by tests/test_oracle_golden.py::test_c_port_* against the reference's ten
 * golden log-likelihoods and against the numpy oracle.
 */
#define _GNU_SOURCE
#include <math.h>
#include <pthread.h>
#include <sched.h>
#include <stdatomic.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

/* Sense-reversing spin barrier (pause, then yield): a likelihood evaluation is a handful of jobs a few milliseconds long,
 * and a futex-based pthread_barrier with ~100 waiters costs as much as a job on a busy host. */
typedef struct { atomic_int count; atomic_int sense; int n; } SpinBarrier;
static void sb_init(SpinBarrier* b, int n) { atomic_init(&b->count, 0); atomic_init(&b->sense, 0); b->n = n; }
static void sb_wait(SpinBarrier* b, int* localSense) {
    *localSense = !*localSense;
    if (atomic_fetch_add_explicit(&b->count, 1, memory_order_acq_rel) == b->n - 1) {
        atomic_store_explicit(&b->count, 0, memory_order_relaxed);
        atomic_store_explicit(&b->sense, *localSense, memory_order_release);
    } else {
        int spins = 0;
        while (atomic_load_explicit(&b->sense, memory_order_acquire) != *localSense) {
#if defined(__x86_64__)
            __builtin_ia32_pause();
#endif
            if (++spins > 20000) { sched_yield(); spins = 0; }
        }
    }
}

typedef struct {
    int tipCount, nBuffers, S, P, nEigen, nMatrices, C, nScale, threads, logScalers;
    double** partials;   /* [nBuffers] -> [C][P][S] or NULL */
    int** states;        /* [nBuffers] -> [P] or NULL */
    double* eigen;       /* [nEigen][2*S*S + S] */
    double* matrices;    /* [nMatrices][C][S][S] row-major (parent i, child j) */
    double* scale;       /* [nScale][P] */
    double* rates;       /* [C] */
    double* weights;     /* [C] */
    double* freqs;       /* [S] */
    double* patternWeights;
    double* site;
    /* persistent worker pool (threads-1 workers + the caller), two barriers per job */
    pthread_t* workers;
    SpinBarrier startBar, endBar;
    int callerSense[2];
    int poolReady, quit, jobKind;
    /* job arguments */
    const int* jobOps; int jobNOps, jobCum;
    int jobEigen; const int* jobProb; const double* jobLen; int jobCount;
} OracleCpu;

typedef struct { OracleCpu* o; int tid; } WorkerArg;
static void run_job(OracleCpu* o, int tid);

static void* worker_main(void* arg) {
    WorkerArg* w = (WorkerArg*)arg;
    OracleCpu* o = w->o;
    const int tid = w->tid;
    free(w);
    /* one worker per hardware thread, pinned: the pattern block a thread owns stays on the NUMA node that first touched
     * it (the partials are first written inside the walk, by the owning thread).  Pin within the CPUs this process may
     * run on: pinning to CPU ids outside that set stacks spinning workers on the same few cores, and every spin barrier
     * then waits for descheduled threads */
    cpu_set_t allowed;
    if (sched_getaffinity(0, sizeof allowed, &allowed) == 0 && o->threads <= CPU_COUNT(&allowed)) {
        int k = tid % CPU_COUNT(&allowed);
        for (int c = 0; c < CPU_SETSIZE; ++c) {
            if (!CPU_ISSET(c, &allowed) || k-- > 0) continue;
            cpu_set_t set;
            CPU_ZERO(&set);
            CPU_SET(c, &set);
            pthread_setaffinity_np(pthread_self(), sizeof set, &set);
            break;
        }
    }
    int s0 = 0, s1 = 0;
    for (;;) {
        sb_wait(&o->startBar, &s0);
        if (o->quit) break;
        run_job(o, tid);
        sb_wait(&o->endBar, &s1);
    }
    return NULL;
}

static void pool_run(OracleCpu* o, int kind) {
    if (o->threads <= 1) { o->jobKind = kind; run_job(o, 0); return; }
    if (!o->poolReady) {
        sb_init(&o->startBar, o->threads);
        sb_init(&o->endBar, o->threads);
        o->callerSense[0] = o->callerSense[1] = 0;
        o->workers = (pthread_t*)malloc(sizeof(pthread_t) * o->threads);
        for (int t = 1; t < o->threads; ++t) {
            WorkerArg* w = (WorkerArg*)malloc(sizeof(WorkerArg));
            w->o = o; w->tid = t;
            pthread_create(&o->workers[t], NULL, worker_main, w);
        }
        o->poolReady = 1;
    }
    o->jobKind = kind;
    sb_wait(&o->startBar, &o->callerSense[0]);
    run_job(o, 0);
    sb_wait(&o->endBar, &o->callerSense[1]);
}

#define EXPORT __attribute__((visibility("default")))

EXPORT OracleCpu* oc_create(int tipCount, int nBuffers, int S, int P, int nEigen, int nMatrices, int C, int nScale,
                            int threads, int logScalers) {
    OracleCpu* o = (OracleCpu*)calloc(1, sizeof(OracleCpu));
    o->tipCount = tipCount; o->nBuffers = nBuffers; o->S = S; o->P = P; o->nEigen = nEigen;
    o->nMatrices = nMatrices; o->C = C; o->nScale = nScale; o->threads = threads < 1 ? 1 : threads;
    o->logScalers = logScalers;
    o->partials = (double**)calloc(nBuffers, sizeof(double*));
    o->states = (int**)calloc(nBuffers, sizeof(int*));
    o->eigen = (double*)calloc((size_t)(nEigen > 0 ? nEigen : 1) * (2 * S * S + S), sizeof(double));
    o->matrices = (double*)calloc((size_t)nMatrices * C * S * S, sizeof(double));
    o->scale = (double*)calloc((size_t)(nScale > 0 ? nScale : 1) * P, sizeof(double));
    o->rates = (double*)calloc(C, sizeof(double));
    o->weights = (double*)calloc(C, sizeof(double));
    o->freqs = (double*)calloc(S, sizeof(double));
    o->patternWeights = (double*)calloc(P, sizeof(double));
    o->site = (double*)calloc(P, sizeof(double));
    for (int c = 0; c < C; ++c) o->rates[c] = 1.0;
    for (int p = 0; p < P; ++p) o->patternWeights[p] = 1.0;
    return o;
}

EXPORT void oc_free(OracleCpu* o) {
    if (o->poolReady) {
        o->quit = 1;
        sb_wait(&o->startBar, &o->callerSense[0]);
        for (int t = 1; t < o->threads; ++t) pthread_join(o->workers[t], NULL);
        free(o->workers);
    }
    for (int b = 0; b < o->nBuffers; ++b) { free(o->partials[b]); free(o->states[b]); }
    free(o->partials); free(o->states); free(o->eigen); free(o->matrices); free(o->scale); free(o->rates);
    free(o->weights); free(o->freqs); free(o->patternWeights); free(o->site); free(o);
}

static double* ensure(OracleCpu* o, int b) {
    if (!o->partials[b]) o->partials[b] = (double*)calloc((size_t)o->C * o->P * o->S, sizeof(double));
    return o->partials[b];
}

EXPORT void oc_set_tip_states(OracleCpu* o, int tip, const int* s) {
    if (!o->states[tip]) o->states[tip] = (int*)malloc(sizeof(int) * o->P);
    memcpy(o->states[tip], s, sizeof(int) * o->P);
    free(o->partials[tip]); o->partials[tip] = NULL;
}
EXPORT void oc_set_partials(OracleCpu* o, int b, const double* x) {
    memcpy(ensure(o, b), x, sizeof(double) * o->C * o->P * o->S);
    free(o->states[b]); o->states[b] = NULL;
}
EXPORT void oc_get_partials(OracleCpu* o, int b, double* x) { memcpy(x, o->partials[b], sizeof(double) * o->C * o->P * o->S); }
EXPORT void oc_set_pattern_weights(OracleCpu* o, const double* w) { memcpy(o->patternWeights, w, sizeof(double) * o->P); }
EXPORT void oc_set_category_rates(OracleCpu* o, const double* r) { memcpy(o->rates, r, sizeof(double) * o->C); }
EXPORT void oc_set_category_weights(OracleCpu* o, const double* w) { memcpy(o->weights, w, sizeof(double) * o->C); }
EXPORT void oc_set_state_frequencies(OracleCpu* o, const double* f) { memcpy(o->freqs, f, sizeof(double) * o->S); }
EXPORT void oc_set_eigen(OracleCpu* o, int idx, const double* evec, const double* ievc, const double* eval) {
    const int S = o->S;
    double* e = o->eigen + (size_t)idx * (2 * S * S + S);
    memcpy(e, evec, sizeof(double) * S * S);
    memcpy(e + S * S, ievc, sizeof(double) * S * S);
    memcpy(e + 2 * S * S, eval, sizeof(double) * S);
}

/* BaseSubstitutionModel.java:206-241; branches [b0,b1) */
static void matrices_range(OracleCpu* o, int b0, int b1) {
    const int S = o->S, C = o->C;
    const double* evec = o->eigen + (size_t)o->jobEigen * (2 * S * S + S);
    const double* ievc = evec + S * S;
    const double* eval = ievc + S * S;
    double* iexp = (double*)malloc(sizeof(double) * S * S);
    for (int b = b0; b < b1; ++b)
        for (int c = 0; c < C; ++c) {
            const double d = o->jobLen[b] * o->rates[c];
            for (int i = 0; i < S; ++i) {
                const double t = exp(d * eval[i]);
                for (int j = 0; j < S; ++j) iexp[i * S + j] = ievc[i * S + j] * t;
            }
            double* m = o->matrices + ((size_t)o->jobProb[b] * C + c) * S * S;
            for (int i = 0; i < S; ++i)
                for (int j = 0; j < S; ++j) {
                    double t = 0.0;
                    for (int k = 0; k < S; ++k) t += evec[i * S + k] * iexp[k * S + j];
                    m[i * S + j] = fabs(t);
                }
        }
    free(iexp);
}

EXPORT void oc_update_transition_matrices(OracleCpu* o, int eigenIdx, const int* probIdx, const double* lengths, int count) {
    o->jobEigen = eigenIdx; o->jobProb = probIdx; o->jobLen = lengths; o->jobCount = count;
    pool_run(o, 1);
}

typedef struct { OracleCpu* o; const int* ops; int nOps, cum, p0, p1; } WalkJob;

static void child_term(const OracleCpu* o, int buf, int mat, int c, int p, double* out) {
    const int S = o->S;
    const double* M = o->matrices + ((size_t)mat * o->C + c) * S * S;
    if (o->states[buf]) {
        const int s = o->states[buf][p];
        if (s < S) for (int i = 0; i < S; ++i) out[i] = M[i * S + s];
        else for (int i = 0; i < S; ++i) out[i] = 1.0;
    } else {
        const double* x = o->partials[buf] + ((size_t)c * o->P + p) * S;
        for (int i = 0; i < S; ++i) {
            double sum = 0.0;
            for (int j = 0; j < S; ++j) sum += M[i * S + j] * x[j];
            out[i] = sum;
        }
    }
}

/* dest[c][p][:] = (M1_c x1[c][p][:]) * (M2_c x2[c][p][:]) for the patterns [p0, p1): the same arithmetic as the scalar
 * statement of GeneralLikelihoodCore.java:171-203 with the four parent states of a cell held in one vector
 * (u = M[:,0] x0 + M[:,1] x1 + M[:,2] x2 + M[:,3] x3).  target_clones: the binary is built once and travels to another
 * host, so the instruction set is picked at load time. */
typedef double v4d __attribute__((vector_size(32), aligned(8)));
__attribute__((target_clones("avx2,fma", "default")))
static void walk4_op(const OracleCpu* o, const int* op, double* dest, int p0, int p1) {
    const int C = o->C, P = o->P;
    for (int c = 0; c < C; ++c) {
        const double* M1 = o->matrices + ((size_t)op[4] * C + c) * 16;
        const double* M2 = o->matrices + ((size_t)op[6] * C + c) * 16;
        v4d a[5], b[5];                                  /* columns of the two matrices; column 4 = gap (all ones) */
        for (int j = 0; j < 4; ++j) {
            a[j] = (v4d){M1[j], M1[4 + j], M1[8 + j], M1[12 + j]};
            b[j] = (v4d){M2[j], M2[4 + j], M2[8 + j], M2[12 + j]};
        }
        a[4] = b[4] = (v4d){1.0, 1.0, 1.0, 1.0};
        const int* s1 = o->states[op[3]];
        const int* s2 = o->states[op[5]];
        const double* x1 = s1 ? NULL : o->partials[op[3]] + (size_t)c * P * 4;
        const double* x2 = s2 ? NULL : o->partials[op[5]] + (size_t)c * P * 4;
        double* d = dest + (size_t)c * P * 4;
        if (!s1 && !s2) {
            for (int p = p0; p < p1; ++p) {
                const double* x = x1 + 4 * p;
                const double* y = x2 + 4 * p;
                const v4d u = a[0] * x[0] + a[1] * x[1] + a[2] * x[2] + a[3] * x[3];
                const v4d v = b[0] * y[0] + b[1] * y[1] + b[2] * y[2] + b[3] * y[3];
                *(v4d*)(d + 4 * p) = u * v;
            }
        } else if (s1 && s2) {
            for (int p = p0; p < p1; ++p) {
                const int sa = s1[p] < 4 ? s1[p] : 4, sb = s2[p] < 4 ? s2[p] : 4;
                *(v4d*)(d + 4 * p) = a[sa] * b[sb];
            }
        } else {
            const int* st = s1 ? s1 : s2;
            const v4d* tc = s1 ? a : b;                  /* tip child's columns */
            const v4d* ic = s1 ? b : a;                  /* internal child's matrix */
            const double* xi = s1 ? x2 : x1;
            for (int p = p0; p < p1; ++p) {
                const double* x = xi + 4 * p;
                const v4d u = ic[0] * x[0] + ic[1] * x[1] + ic[2] * x[2] + ic[3] * x[3];
                *(v4d*)(d + 4 * p) = u * tc[st[p] < 4 ? st[p] : 4];
            }
        }
    }
}

static void* walk_block(void* arg) {
    WalkJob* w = (WalkJob*)arg;
    OracleCpu* o = w->o;
    const int S = o->S, C = o->C, P = o->P;
    double a[256], b[256];
    for (int k = 0; k < w->nOps; ++k) {
        const int* op = w->ops + 7 * k;
        double* dest = o->partials[op[0]];
        if (S == 4) {          /* nucleotide fast path: one 4-state cell = one 256-bit vector (AVX2 + FMA clone) */
            walk4_op(o, op, dest, w->p0, w->p1);
        } else {
            for (int c = 0; c < C; ++c)
                for (int p = w->p0; p < w->p1; ++p) {
                    child_term(o, op[3], op[4], c, p, a);
                    child_term(o, op[5], op[6], c, p, b);
                    double* d = dest + ((size_t)c * P + p) * S;
                    for (int i = 0; i < S; ++i) d[i] = a[i] * b[i];
                }
        }
        if (op[1] >= 0) {      /* AbstractLikelihoodCore.java:406-442, unconditional */
            double* sf = o->scale + (size_t)op[1] * P;
            for (int p = w->p0; p < w->p1; ++p) {
                double m = 0.0;
                for (int c = 0; c < C; ++c) {
                    const double* d = dest + ((size_t)c * P + p) * S;
                    for (int i = 0; i < S; ++i) if (d[i] > m) m = d[i];
                }
                if (m == 0.0) m = 1.0;
                for (int c = 0; c < C; ++c) {
                    double* d = dest + ((size_t)c * P + p) * S;
                    for (int i = 0; i < S; ++i) d[i] /= m;
                }
                const double lm = log(m);
                sf[p] = o->logScalers ? lm : m;
                if (w->cum >= 0) o->scale[(size_t)w->cum * P + p] += lm;
            }
        } else if (op[2] >= 0) {
            const double* sf = o->scale + (size_t)op[2] * P;
            for (int p = w->p0; p < w->p1; ++p) {
                const double f = o->logScalers ? exp(sf[p]) : sf[p];
                for (int c = 0; c < C; ++c) {
                    double* d = dest + ((size_t)c * P + p) * S;
                    for (int i = 0; i < S; ++i) d[i] /= f;
                }
            }
        }
    }
    return NULL;
}

EXPORT void oc_update_partials(OracleCpu* o, const int* ops, int nOps, int cum) {
    for (int k = 0; k < nOps; ++k) {
        ensure(o, ops[7 * k]);
        free(o->states[ops[7 * k]]); o->states[ops[7 * k]] = NULL;
    }
    o->jobOps = ops; o->jobNOps = nOps; o->jobCum = cum;
    pool_run(o, 0);
}

static void split(int n, int T, int tid, int* a, int* b) {
    const int div = n / T, rem = n % T;
    *a = tid * div + (tid < rem ? tid : rem);
    *b = *a + div + (tid < rem ? 1 : 0);
}

static void run_job(OracleCpu* o, int tid) {
    int a, b;
    if (o->jobKind == 0) {
        split(o->P, o->threads, tid, &a, &b);      /* contiguous pattern blocks (Patterns.java:142-169 rule) */
        if (b > a) {
            WalkJob w = {o, o->jobOps, o->jobNOps, o->jobCum, a, b};
            walk_block(&w);
        }
    } else {
        split(o->jobCount, o->threads, tid, &a, &b);
        if (b > a) matrices_range(o, a, b);
    }
}

EXPORT void oc_reset_scale_factors(OracleCpu* o, int cum) { memset(o->scale + (size_t)cum * o->P, 0, sizeof(double) * o->P); }

/* AbstractLikelihoodCore.java:451-459 / BDLD:915-926 */
EXPORT void oc_accumulate_scale_factors(OracleCpu* o, const int* idx, int count, int cum) {
    double* c = o->scale + (size_t)cum * o->P;
    for (int k = 0; k < count; ++k) {
        const double* s = o->scale + (size_t)idx[k] * o->P;
        for (int p = 0; p < o->P; ++p) c[p] += o->logScalers ? s[p] : log(s[p]);
    }
}

/* GeneralLikelihoodCore.java:358-408 */
EXPORT double oc_calculate_root_log_likelihoods(OracleCpu* o, int root, int cum) {
    const int S = o->S, C = o->C, P = o->P;
    const double* r = o->partials[root];
    double total = 0.0;
    for (int p = 0; p < P; ++p) {
        double sum = 0.0;
        for (int i = 0; i < S; ++i) {
            double integ = 0.0;
            for (int c = 0; c < C; ++c) integ += r[((size_t)c * P + p) * S + i] * o->weights[c];
            sum += o->freqs[i] * integ;
        }
        double s = log(sum);
        if (cum >= 0) s += o->scale[(size_t)cum * P + p];
        o->site[p] = s;
        total += o->patternWeights[p] * s;
    }
    return total;
}

EXPORT void oc_get_site_log_likelihoods(OracleCpu* o, double* out) { memcpy(out, o->site, sizeof(double) * o->P); }
EXPORT void oc_get_log_scale_factors(OracleCpu* o, int idx, double* out) {
    const double* s = o->scale + (size_t)idx * o->P;
    for (int p = 0; p < o->P; ++p) out[p] = o->logScalers ? s[p] : log(s[p]);
}
