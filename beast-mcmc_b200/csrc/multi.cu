// multi.cu -- the engine's own multi-GPU layer (SURVEY.md 8e, mode B): ONE BEAGLE instance whose site patterns are
// sharded over several GPUs of the node, so that an unmodified BEAST run (one likelihood, no -beagle_instances) uses
// all of them by naming one resource ("-beagle_order <n+1>" on an n-GPU box, see buildResources in api.cu).
//
//   * sharding rule = the reference's own (-beagle_instances): contiguous blocks, floor(P/g) patterns each, the first
//     P mod g shards one more (src/dr/evolution/alignment/Patterns.java:142-169) -- shard k of a sharded instance holds
//     exactly the patterns BEAST's k-th sub-instance would, so per-shard results are bit-comparable with mode A;
//   * every shard is an ordinary single-device Instance (own stream, own plan cache); calls fan out over a small pool of
//     host threads (one per shard, spin-then-sleep hand-off) so that the g devices are fed concurrently;
//   * the only exchange on the data path is the sum of the g per-shard log-likelihoods: the finishing block of every
//     shard's k_root stores its sum into all members' slot arrays over NVLink peer mappings and adds what the others
//     stored (Exchange in engine.h) -- no NCCL launch, no host arithmetic, one 8-byte D2H of the joint value;
//   * per-pattern outputs (getPartials, getSiteLogLikelihoods, scale factors, per-pattern derivatives) are gathered,
//     per-pattern inputs (tip states / partials, pattern weights) sliced, everything else broadcast.
// *ByPartition calls are not offered on a sharded instance (partitions and pattern shards would have to be composed;
// BEAST's MultiPartitionDataLikelihoodDelegate then takes a single-device resource).
//
// Also here: the reduce-group set-up used by one-process-per-GPU callers (bench.py under torchrun): b200Exchange*.
#include "../../include/libhmsbeagle_b200.h"
#include "engine.h"
#include "multi.h"

#include <atomic>
#include <condition_variable>
#include <cmath>
#include <cstring>
#include <functional>
#include <thread>

namespace b200 {

// ---- host thread pool: one worker per shard beyond the first (the caller drives shard 0) ---------------------------------
class ShardPool {
  public:
    explicit ShardPool(int n) : n_(n), rc_(n, 0) {
        for (int k = 1; k < n; ++k) workers_.emplace_back([this, k] { loop(k); });
    }
    ~ShardPool() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            quit_ = true;
            gen_.fetch_add(1, std::memory_order_release);
        }
        cv_.notify_all();
        for (auto& t : workers_) t.join();
    }
    // run fn(k) for every shard k concurrently; returns the first non-zero result in shard order
    int run(const std::function<int(int)>& fn) {
        if (n_ == 1) return fn(0);
        fn_ = &fn;
        pending_.store(n_ - 1, std::memory_order_relaxed);
        {
            std::lock_guard<std::mutex> lk(mu_);
            gen_.fetch_add(1, std::memory_order_release);
        }
        cv_.notify_all();
        rc_[0] = fn(0);
        for (int spin = 0; pending_.load(std::memory_order_acquire) != 0; ++spin)
            if (spin > 2000) std::this_thread::yield();
        for (int k = 0; k < n_; ++k) if (rc_[k] != 0) return rc_[k];
        return 0;
    }

  private:
    void loop(int k) {
        unsigned long seen = 0;
        for (;;) {
            // short spin (a likelihood evaluation is a burst of calls a few microseconds apart), then sleep
            bool woke = false;
            for (int spin = 0; spin < 20000; ++spin) {
                if (gen_.load(std::memory_order_acquire) != seen) { woke = true; break; }
#if defined(__x86_64__)
                __builtin_ia32_pause();
#endif
            }
            if (!woke) {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return gen_.load(std::memory_order_acquire) != seen; });
            }
            seen = gen_.load(std::memory_order_acquire);
            if (quit_) return;
            rc_[k] = (*fn_)(k);
            pending_.fetch_sub(1, std::memory_order_release);
        }
    }
    int n_;
    std::vector<std::thread> workers_;
    std::vector<int> rc_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::atomic<unsigned long> gen_{0};
    std::atomic<int> pending_{0};
    const std::function<int(int)>* fn_ = nullptr;
    bool quit_ = false;
};

struct Sharded {
    int g = 0, P = 0, S = 0, C = 0, tipCount = 0;
    std::vector<int> child;            // instance ids of the shards
    std::vector<int> begin, count;     // pattern block of every shard
    ShardPool* pool = nullptr;
    bool logScalers = false;
    ~Sharded() { delete pool; }
};

// Patterns.java:142-169: shard k of g gets floor(P/g) patterns, the first P mod g shards one more
static void blockRule(int P, int g, std::vector<int>& begin, std::vector<int>& count) {
    begin.resize(g); count.resize(g);
    int at = 0;
    for (int k = 0; k < g; ++k) {
        count[k] = P / g + (k < P % g ? 1 : 0);
        begin[k] = at;
        at += count[k];
    }
}

// ---- reduce groups ----------------------------------------------------------------------------------------------------------
static int exchangeAllocate(Instance* in, int rank, int size) {
    if (size < 1 || size > kMaxGroup || rank < 0 || rank >= size) return BEAGLE_ERROR_OUT_OF_RANGE;
    if (cudaSetDevice(in->device) != cudaSuccess) return BEAGLE_ERROR_GENERAL;
    if (in->dSlots != nullptr) return BEAGLE_ERROR_GENERAL;            // one group per instance
    const size_t bytes = sizeof(ExchangeSlot) * 2 * size;
    if (cudaMalloc(reinterpret_cast<void**>(&in->dSlots), bytes) != cudaSuccess) { cudaGetLastError(); return BEAGLE_ERROR_OUT_OF_MEMORY; }
    if (cudaMemset(in->dSlots, 0, bytes) != cudaSuccess) return BEAGLE_ERROR_GENERAL;
    in->exchange = Exchange();
    in->exchange.rank = rank;
    in->exchange.size = size;
    in->exchange.seq = 0;
    int clockKHz = 1965000;
    cudaDeviceGetAttribute(&clockKHz, cudaDevAttrClockRate, in->device);
    in->exchange.timeoutCycles = (long long)clockKHz * 1000ll * 4ll;   // ~4 s of SM clocks: a peer that never launches
    in->exchange.peers[rank] = in->dSlots;
    return BEAGLE_SUCCESS;
}

void exchangeRelease(Instance* in) {
    if (in->dSlots == nullptr && in->ipcOpened.empty()) return;
    cudaSetDevice(in->device);
    for (void* p : in->ipcOpened) cudaIpcCloseMemHandle(p);
    in->ipcOpened.clear();
    cudaFree(in->dSlots);
    in->dSlots = nullptr;
    in->exchangeOn = false;
}

}  // namespace b200

using namespace b200;

extern "C" {

// ---- one process per GPU (bench.py under torchrun, or any MPI-style caller) ------------------------------------------------
int b200ExchangeCreate(int instance, int rank, int size, void* outIpcHandle64) {
    Instance* in = instanceById(instance);
    if (in == nullptr) return BEAGLE_ERROR_UNINITIALIZED_INSTANCE;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "the handle travels as 64 opaque bytes");
    int rc = exchangeAllocate(in, rank, size);
    if (rc != BEAGLE_SUCCESS) return rc;
    if (outIpcHandle64 != nullptr) {
        cudaIpcMemHandle_t h;
        if (cudaIpcGetMemHandle(&h, in->dSlots) != cudaSuccess) { cudaGetLastError(); return BEAGLE_ERROR_GENERAL; }
        memcpy(outIpcHandle64, &h, 64);
    }
    return BEAGLE_SUCCESS;
}

int b200ExchangeConnect(int instance, const void* allIpcHandles64) {
    Instance* in = instanceById(instance);
    if (in == nullptr || in->dSlots == nullptr) return BEAGLE_ERROR_UNINITIALIZED_INSTANCE;
    if (cudaSetDevice(in->device) != cudaSuccess) return BEAGLE_ERROR_GENERAL;
    const char* all = static_cast<const char*>(allIpcHandles64);
    for (int q = 0; q < in->exchange.size; ++q) {
        if (q == in->exchange.rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, all + 64 * (size_t)q, 64);
        void* mapped = nullptr;
        if (cudaIpcOpenMemHandle(&mapped, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
            cudaGetLastError();
            return BEAGLE_ERROR_NO_RESOURCE;                            // no peer path between the two devices
        }
        in->ipcOpened.push_back(mapped);
        in->exchange.peers[q] = static_cast<ExchangeSlot*>(mapped);
    }
    in->exchangeOn = in->exchange.size > 1;
    return BEAGLE_SUCCESS;
}

// ---- several instances of ONE process (what a JVM holds): peer mappings instead of IPC --------------------------------------
int b200ExchangeConnectLocal(const int* instances, int count) {
    if (count < 1 || count > kMaxGroup) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<Instance*> m(count);
    for (int k = 0; k < count; ++k) {
        m[k] = instanceById(instances[k]);
        if (m[k] == nullptr) return BEAGLE_ERROR_UNINITIALIZED_INSTANCE;
    }
    for (int k = 0; k < count; ++k) {
        int rc = exchangeAllocate(m[k], k, count);
        if (rc != BEAGLE_SUCCESS) return rc;
    }
    for (int k = 0; k < count; ++k) {
        if (cudaSetDevice(m[k]->device) != cudaSuccess) return BEAGLE_ERROR_GENERAL;
        for (int q = 0; q < count; ++q) {
            if (m[q]->device != m[k]->device) {
                int can = 0;
                cudaDeviceCanAccessPeer(&can, m[k]->device, m[q]->device);
                if (!can) return BEAGLE_ERROR_NO_RESOURCE;
                cudaError_t e = cudaDeviceEnablePeerAccess(m[q]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return BEAGLE_ERROR_NO_RESOURCE; }
                cudaGetLastError();
            }
            m[k]->exchange.peers[q] = m[q]->dSlots;
        }
        m[k]->exchangeOn = count > 1;
    }
    return BEAGLE_SUCCESS;
}

}  // extern "C"

// =====================================================================================================================
// sharded instance
// =====================================================================================================================
namespace b200 {

int shardedCreate(Instance* parent, int g, const int* devices, int tipCount, int partialsBufferCount, int compactBufferCount,
                  int stateCount, int patternCount, int eigenBufferCount, int matrixBufferCount, int categoryCount,
                  int scaleBufferCount, long preferenceFlags, long requirementFlags, void* detailsOut) {
    BeagleInstanceDetails* details = static_cast<BeagleInstanceDetails*>(detailsOut);
    Sharded* sh = new Sharded();
    sh->g = g; sh->P = patternCount; sh->S = stateCount; sh->C = categoryCount; sh->tipCount = tipCount;
    sh->logScalers = (requirementFlags | preferenceFlags) & BEAGLE_FLAG_SCALERS_LOG;
    blockRule(patternCount, g, sh->begin, sh->count);
    for (int k = 0; k < g; ++k) {
        int res[1] = {devices[k] + 1};
        BeagleInstanceDetails d{};
        const int id = beagleCreateInstance(tipCount, partialsBufferCount, compactBufferCount, stateCount,
                                            std::max(1, sh->count[k]), eigenBufferCount, matrixBufferCount, categoryCount,
                                            scaleBufferCount, res, 1, preferenceFlags, requirementFlags, &d);
        if (id < 0) {
            for (int c : sh->child) beagleFinalizeInstance(c);
            delete sh;
            return id;
        }
        sh->child.push_back(id);
        if (k == 0) parent->flags = d.flags;        // the shards' negotiated flags (precision included)
        if (k == 0 && details != nullptr) *details = d;
    }
    if (g > 1) {
        const int rc = b200ExchangeConnectLocal(sh->child.data(), g);
        if (rc != BEAGLE_SUCCESS) {
            for (int c : sh->child) beagleFinalizeInstance(c);
            delete sh;
            return rc;
        }
    }
    // a shard without patterns (P < g) keeps one padded pattern of weight zero and takes part in the exchange with sum 0
    for (int k = 0; k < g; ++k)
        if (sh->count[k] == 0) { const double zero = 0.0; beagleSetPatternWeights(sh->child[k], &zero); }
    sh->pool = new ShardPool(g);
    parent->shard = sh;
    return BEAGLE_SUCCESS;
}

void shardedDestroy(Instance* parent) {
    Sharded* sh = static_cast<Sharded*>(parent->shard);
    if (sh == nullptr) return;
    for (int c : sh->child) beagleFinalizeInstance(c);
    delete sh;
    parent->shard = nullptr;
}

namespace {
inline int nz(const Sharded* sh, int k) { return std::max(1, sh->count[k]); }      // pattern count the shard was created with

// per-pattern double array [P] -> shard block
int slicePerPattern(Sharded* sh, const double* in, const std::function<int(int, const double*)>& call) {
    return sh->pool->run([&](int k) {
        if (sh->count[k] == 0) return 0;
        return call(sh->child[k], in + sh->begin[k]);
    });
}
}  // namespace

int shSetTipStates(Sharded* sh, int tip, const int* states) {
    return sh->pool->run([&](int k) {
        if (sh->count[k] == 0) { int gap = sh->S; return beagleSetTipStates(sh->child[k], tip, &gap); }
        return beagleSetTipStates(sh->child[k], tip, states + sh->begin[k]);
    });
}

int shGetTipStates(Sharded* sh, int tip, int* states) {
    return sh->pool->run([&](int k) {
        if (sh->count[k] == 0) return 0;
        return beagleGetTipStates(sh->child[k], tip, states + sh->begin[k]);
    });
}

// [C or 1][P][S] -> [C or 1][P_k][S]
int shSetPartials(Sharded* sh, int buffer, const double* in, bool perCategory) {
    const int reps = perCategory ? sh->C : 1;
    return sh->pool->run([&](int k) {
        const int n = nz(sh, k);
        std::vector<double> part((size_t)reps * n * sh->S, 1.0);
        for (int c = 0; c < reps; ++c)
            if (sh->count[k] > 0)
                memcpy(part.data() + (size_t)c * n * sh->S, in + ((size_t)c * sh->P + sh->begin[k]) * sh->S,
                       sizeof(double) * (size_t)sh->count[k] * sh->S);
        return perCategory ? beagleSetPartials(sh->child[k], buffer, part.data())
                           : beagleSetTipPartials(sh->child[k], buffer, part.data());
    });
}

int shGetPartials(Sharded* sh, int buffer, int scaleIndex, double* out) {
    return sh->pool->run([&](int k) {
        const int n = nz(sh, k);
        std::vector<double> part((size_t)sh->C * n * sh->S);
        const int rc = beagleGetPartials(sh->child[k], buffer, scaleIndex, part.data());
        if (rc != 0 || sh->count[k] == 0) return rc;
        for (int c = 0; c < sh->C; ++c)
            memcpy(out + ((size_t)c * sh->P + sh->begin[k]) * sh->S, part.data() + (size_t)c * n * sh->S,
                   sizeof(double) * (size_t)sh->count[k] * sh->S);
        return 0;
    });
}

int shSetPatternWeights(Sharded* sh, const double* w) {
    return slicePerPattern(sh, w, [](int id, const double* p) { return beagleSetPatternWeights(id, p); });
}

int shBroadcast(Sharded* sh, const std::function<int(int)>& call) {
    return sh->pool->run([&](int k) { return call(sh->child[k]); });
}

int shGetPerPattern(Sharded* sh, double* out, const std::function<int(int, double*)>& call) {
    return sh->pool->run([&](int k) {
        std::vector<double> part(nz(sh, k));
        const int rc = call(sh->child[k], part.data());
        if (rc == 0 && sh->count[k] > 0) memcpy(out + sh->begin[k], part.data(), sizeof(double) * sh->count[k]);
        return rc;
    });
}

// every shard launches its k_root with the exchange; the joint value is read from shard 0 (all members hold the same)
int shRoot(Sharded* sh, const int* bufferIndices, const int* wIdx, const int* fIdx, const int* cumIdx, int count, double* out) {
    if (count != 1) return BEAGLE_ERROR_NO_IMPLEMENTATION;
    std::vector<double> joint(sh->g, 0.0);
    const int rc = sh->pool->run([&](int k) {
        const int r = beagleCalculateRootLogLikelihoods(sh->child[k], bufferIndices, wIdx, fIdx, cumIdx, 1, &joint[k]);
        return r == BEAGLE_ERROR_FLOATING_POINT ? 0 : r;
    });
    if (rc != 0) return rc;
    *out = joint[0];
    return std::isnan(joint[0]) ? BEAGLE_ERROR_FLOATING_POINT : BEAGLE_SUCCESS;
}

int shEdgeDerivatives(Sharded* sh, const int* post, const int* pre, const int* dmat, const int* wIdx, int count, double* outPer,
                      double* outSum, double* outSumSq) {
    std::vector<std::vector<double>> per(sh->g), s1(sh->g), s2(sh->g);
    const int rc = sh->pool->run([&](int k) {
        if (outPer) per[k].resize((size_t)count * nz(sh, k));
        s1[k].assign(count, 0.0); s2[k].assign(count, 0.0);
        return beagleCalculateEdgeDerivatives(sh->child[k], post, pre, dmat, wIdx, count, outPer ? per[k].data() : nullptr,
                                              s1[k].data(), s2[k].data());
    });
    if (rc != 0) return rc;
    for (int e = 0; e < count; ++e) {
        double a = 0.0, b = 0.0;
        for (int k = 0; k < sh->g; ++k) { if (sh->count[k] == 0) continue; a += s1[k][e]; b += s2[k][e]; }
        if (outSum) outSum[e] = a;
        if (outSumSq) outSumSq[e] = b;
        if (outPer)
            for (int k = 0; k < sh->g; ++k)
                if (sh->count[k] > 0)
                    memcpy(outPer + (size_t)e * sh->P + sh->begin[k], per[k].data() + (size_t)e * nz(sh, k),
                           sizeof(double) * sh->count[k]);
    }
    return BEAGLE_SUCCESS;
}

// every shard samples its block with the GLOBAL pattern index in the Philox counter: the draws equal the unsharded instance's
int shSampleAncestralStates(Sharded* sh, const int* nodeBuffers, const int* parentRows, const int* matrixIndices, int count,
                            int rootBuffer, int wIdx, int fIdx, unsigned long long seed, unsigned long long drawIndex,
                            int* outStates, int* outCategories) {
    if (count < 1 || outStates == nullptr || outCategories == nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<std::vector<int>> states(sh->g), cats(sh->g);
    const int rc = sh->pool->run([&](int k) {
        if (sh->count[k] == 0) return 0;
        states[k].resize((size_t)count * sh->count[k]);
        cats[k].resize(sh->count[k]);
        return sampleAncestralStates(sh->child[k], nodeBuffers, parentRows, matrixIndices, count, rootBuffer, wIdx, fIdx, seed,
                                     drawIndex, sh->begin[k], states[k].data(), cats[k].data());
    });
    if (rc != 0) return rc;
    for (int k = 0; k < sh->g; ++k) {
        if (sh->count[k] == 0) continue;
        memcpy(outCategories + sh->begin[k], cats[k].data(), sizeof(int) * sh->count[k]);
        for (int r = 0; r < count; ++r)
            memcpy(outStates + (size_t)r * sh->P + sh->begin[k], states[k].data() + (size_t)r * sh->count[k],
                   sizeof(int) * sh->count[k]);
    }
    return BEAGLE_SUCCESS;
}

// as shSampleAncestralStates; the shards' branch totals are added on the host in shard order
int shSampleMarkovJumps(Sharded* sh, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                        const double* edgeLengths, int count, int rootBuffer, int wIdx, int fIdx, int eigenIndex, int rIdx,
                        const double* registerMatrices, int registerCount, unsigned long long seed, unsigned long long drawIndex,
                        int* outStates, int* outCategories, double* outBranchCounts, double* outPatternCounts) {
    if (count < 1 || registerCount < 1 || registerCount > kMaxJumpRegisters) return BEAGLE_ERROR_OUT_OF_RANGE;
    const size_t G = registerCount;
    std::vector<std::vector<int>> states(sh->g), cats(sh->g);
    std::vector<std::vector<double>> branch(sh->g), pattern(sh->g);
    const int rc = sh->pool->run([&](int k) {
        const size_t n = sh->count[k];
        if (n == 0) return 0;
        if (outStates != nullptr) states[k].resize((size_t)count * n);
        if (outCategories != nullptr) cats[k].resize(n);
        if (outBranchCounts != nullptr) branch[k].resize(G * count);
        if (outPatternCounts != nullptr) pattern[k].resize(G * n);
        auto ptr = [](auto& v) { return v.empty() ? nullptr : v.data(); };
        return sampleMarkovJumps(sh->child[k], nodeBuffers, parentRows, matrixIndices, edgeLengths, count, rootBuffer, wIdx,
                                 fIdx, eigenIndex, rIdx, registerMatrices, registerCount, seed, drawIndex, sh->begin[k],
                                 ptr(states[k]), ptr(cats[k]), ptr(branch[k]), ptr(pattern[k]));
    });
    if (rc != 0) return rc;
    if (outBranchCounts != nullptr) std::fill(outBranchCounts, outBranchCounts + G * count, 0.0);
    for (int k = 0; k < sh->g; ++k) {
        const size_t n = sh->count[k];
        if (n == 0) continue;
        if (outCategories != nullptr) memcpy(outCategories + sh->begin[k], cats[k].data(), sizeof(int) * n);
        if (outStates != nullptr)
            for (int r = 0; r < count; ++r)
                memcpy(outStates + (size_t)r * sh->P + sh->begin[k], states[k].data() + (size_t)r * n, sizeof(int) * n);
        if (outBranchCounts != nullptr) for (size_t q = 0; q < G * count; ++q) outBranchCounts[q] += branch[k][q];
        if (outPatternCounts != nullptr)
            for (size_t g = 0; g < G; ++g)
                memcpy(outPatternCounts + g * sh->P + sh->begin[k], pattern[k].data() + g * n, sizeof(double) * n);
    }
    return BEAGLE_SUCCESS;
}

// as shSampleMarkovJumps.  Round 1 gives every shard's fixed-size outputs, jump counts and event total; when events are
// asked for and the total over all shards fits eventCapacity, round 2 draws each shard's events, and they are reassembled in
// global (row, pattern) order from the shards' jump counts.
int shSampleSubstitutionHistories(Sharded* sh, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                                  const double* edgeLengths, int count, int rootBuffer, int wIdx, int fIdx, int rIdx,
                                  const double* rateMatrix, const double* registerMatrices, int registerCount,
                                  unsigned long long seed, unsigned long long drawIndex, int* outStates, int* outCategories,
                                  double* outBranchCounts, double* outPatternCounts, int* outJumpCounts, long long eventCapacity,
                                  long long* outEventCount, double* outEventTimes, int* outEventStates) {
    double mu = 0.0;
    if (count < 1) return BEAGLE_ERROR_OUT_OF_RANGE;
    int rc = checkHistoryArguments(sh->S, rateMatrix, registerCount, eventCapacity, outEventCount, outEventTimes,
                                   outEventStates, &mu);
    if (rc != BEAGLE_SUCCESS) return rc;
    const bool wantEvents = outEventTimes != nullptr || outEventStates != nullptr;
    const size_t G = registerCount;
    std::vector<std::vector<int>> states(sh->g), cats(sh->g), jumps(sh->g), evStates(sh->g);
    std::vector<std::vector<double>> branch(sh->g), pattern(sh->g), evTimes(sh->g);
    std::vector<long long> events(sh->g, 0);
    auto ptr = [](auto& v) { return v.empty() ? nullptr : v.data(); };
    rc = sh->pool->run([&](int k) {
        const size_t n = sh->count[k];
        if (n == 0) return 0;
        if (outStates != nullptr) states[k].resize((size_t)count * n);
        if (outCategories != nullptr) cats[k].resize(n);
        if (outBranchCounts != nullptr) branch[k].resize(G * count);
        if (outPatternCounts != nullptr) pattern[k].resize(G * n);
        if (outJumpCounts != nullptr || wantEvents) jumps[k].resize((size_t)count * n);
        return sampleSubstitutionHistories(sh->child[k], nodeBuffers, parentRows, matrixIndices, edgeLengths, count, rootBuffer,
                                           wIdx, fIdx, rIdx, rateMatrix, registerMatrices, registerCount, seed, drawIndex,
                                           sh->begin[k], ptr(states[k]), ptr(cats[k]), ptr(branch[k]), ptr(pattern[k]),
                                           ptr(jumps[k]), 0, outEventCount != nullptr ? &events[k] : nullptr, nullptr, nullptr);
    });
    if (rc != 0) return rc;
    long long total = 0;
    for (int k = 0; k < sh->g; ++k) total += events[k];
    const bool fits = total <= eventCapacity;
    if (wantEvents && fits && total > 0) {
        rc = sh->pool->run([&](int k) {
            if (sh->count[k] == 0 || events[k] == 0) return 0;
            if (outEventTimes != nullptr) evTimes[k].resize(events[k]);
            if (outEventStates != nullptr) evStates[k].resize(events[k]);
            long long got = 0;
            return sampleSubstitutionHistories(sh->child[k], nodeBuffers, parentRows, matrixIndices, edgeLengths, count,
                                               rootBuffer, wIdx, fIdx, rIdx, rateMatrix, registerMatrices, registerCount, seed,
                                               drawIndex, sh->begin[k], nullptr, nullptr, nullptr, nullptr, nullptr, events[k],
                                               &got, ptr(evTimes[k]), ptr(evStates[k]));
        });
        if (rc != 0) return rc;
        std::vector<long long> pos(sh->g, 0);                    // next event of each shard
        long long out = 0;
        for (int r = 0; r < count; ++r)
            for (int k = 0; k < sh->g; ++k) {
                const size_t n = sh->count[k];
                long long m = 0;
                for (size_t p = 0; p < n; ++p) m += jumps[k][(size_t)r * n + p];
                if (outEventTimes != nullptr)
                    memcpy(outEventTimes + out, evTimes[k].data() + pos[k], sizeof(double) * m);
                if (outEventStates != nullptr)
                    memcpy(outEventStates + out, evStates[k].data() + pos[k], sizeof(int) * m);
                pos[k] += m;
                out += m;
            }
    }
    if (outBranchCounts != nullptr) std::fill(outBranchCounts, outBranchCounts + G * count, 0.0);
    for (int k = 0; k < sh->g; ++k) {
        const size_t n = sh->count[k];
        if (n == 0) continue;
        if (outCategories != nullptr) memcpy(outCategories + sh->begin[k], cats[k].data(), sizeof(int) * n);
        for (int r = 0; r < count; ++r) {
            if (outStates != nullptr)
                memcpy(outStates + (size_t)r * sh->P + sh->begin[k], states[k].data() + (size_t)r * n, sizeof(int) * n);
            if (outJumpCounts != nullptr)
                memcpy(outJumpCounts + (size_t)r * sh->P + sh->begin[k], jumps[k].data() + (size_t)r * n, sizeof(int) * n);
        }
        if (outBranchCounts != nullptr) for (size_t q = 0; q < G * count; ++q) outBranchCounts[q] += branch[k][q];
        if (outPatternCounts != nullptr)
            for (size_t g = 0; g < G; ++g)
                memcpy(outPatternCounts + g * sh->P + sh->begin[k], pattern[k].data() + g * n, sizeof(double) * n);
    }
    if (outEventCount != nullptr) *outEventCount = total;
    return wantEvents && !fits ? BEAGLE_ERROR_OUT_OF_RANGE : BEAGLE_SUCCESS;
}

int shCrossProducts(Sharded* sh, const int* post, const int* pre, const int* rIdx, const int* wIdx, const double* lengths,
                    int count, double* outSum, double* outSumSq) {
    if (outSumSq != nullptr) return BEAGLE_ERROR_NO_IMPLEMENTATION;
    const size_t n = (size_t)sh->S * sh->S;
    std::vector<std::vector<double>> acc(sh->g);
    const int rc = sh->pool->run([&](int k) {
        acc[k].assign(n, 0.0);
        if (sh->count[k] == 0) return 0;
        return beagleCalculateCrossProductDerivative(sh->child[k], post, pre, rIdx, wIdx, lengths, count, acc[k].data(), nullptr);
    });
    if (rc != 0) return rc;
    for (int k = 0; k < sh->g; ++k)
        for (size_t q = 0; q < n; ++q) outSum[q] += acc[k][q];
    return BEAGLE_SUCCESS;
}

}  // namespace b200
