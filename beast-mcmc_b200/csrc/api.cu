// api.cu -- the C ABI of libhmsbeagle.so (declared in include/libhmsbeagle_b200.h).
//
// Host side of the engine: instance table, resource list, buffer bookkeeping, translation of the
// caller's integer op tuples into device op records (with dependency-safe re-ordering and operand
// stack-slot assignment), and stream-ordered launches.  Every entry point selects the instance's
// device explicitly: JNI calls arrive from arbitrary pool threads (CompoundLikelihood.java:63-75).
// There is NO CPU fallback: without a CUDA device beagleCreateInstance fails with
// BEAGLE_ERROR_NO_RESOURCE.
#include "../../include/libhmsbeagle_b200.h"
#include "engine.h"
#include "multi.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>

using namespace b200;

namespace {

std::mutex gMutex;
std::vector<Instance*> gInstances;

const long kSupportedFlags =
    BEAGLE_FLAG_PRECISION_DOUBLE | BEAGLE_FLAG_PRECISION_SINGLE | BEAGLE_FLAG_COMPUTATION_SYNCH | BEAGLE_FLAG_EIGEN_REAL |
    BEAGLE_FLAG_EIGEN_COMPLEX | BEAGLE_FLAG_SCALING_MANUAL | BEAGLE_FLAG_SCALING_DYNAMIC |
    BEAGLE_FLAG_SCALERS_RAW | BEAGLE_FLAG_SCALERS_LOG | BEAGLE_FLAG_VECTOR_NONE | BEAGLE_FLAG_THREADING_NONE |
    BEAGLE_FLAG_PROCESSOR_GPU | BEAGLE_FLAG_FRAMEWORK_CUDA | BEAGLE_FLAG_PARALLELOPS_GRID |
    BEAGLE_FLAG_PREORDER_TRANSPOSE_AUTO;     // updatePrePartials always applies the node matrix transposed itself

int envInt(const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
}

int flushPending(Instance* in);

Instance* getInstance(int id) {
    std::lock_guard<std::mutex> lock(gMutex);
    if (id < 0 || id >= (int)gInstances.size()) return nullptr;
    return gInstances[id];
}

// a pattern-sharded instance forwards every call to its shards (multi.cu); SH(expr) runs at the top of an entry point
#define SH(id, expr)                                                                         \
    do {                                                                                     \
        Instance* p__ = getInstance(id);                                                     \
        if (p__ != nullptr && p__->shard != nullptr) {                                       \
            Sharded* sh = static_cast<Sharded*>(p__->shard);                                 \
            (void)sh;                                                                        \
            return (expr);                                                                   \
        }                                                                                    \
    } while (0)

// GET_INSTANCE_LAZY: the three calls of a deferred small evaluation (incr.cu) manage the pending work themselves;
// GET_INSTANCE: every other entry point first launches whatever was deferred, so that it observes completed semantics
#define GET_INSTANCE_LAZY(in, id)                                       \
    Instance* in = getInstance(id);                                     \
    if (in == nullptr) return BEAGLE_ERROR_UNINITIALIZED_INSTANCE;      \
    if (in->shard != nullptr) return BEAGLE_ERROR_NO_IMPLEMENTATION;    \
    if (cudaSetDevice(in->device) != cudaSuccess) return BEAGLE_ERROR_GENERAL;

#define GET_INSTANCE(in, id)                                            \
    GET_INSTANCE_LAZY(in, id)                                           \
    if (!in->pendingMats.empty() || !in->pendingOps.empty()) {          \
        const int flushRc__ = flushPending(in);                         \
        if (flushRc__ != BEAGLE_SUCCESS) return flushRc__;              \
    }

#define CUDA_OK(expr)                                                                        \
    do {                                                                                     \
        cudaError_t e__ = (expr);                                                            \
        if (e__ != cudaSuccess) {                                                            \
            if (getenv("B200_BEAGLE_DEBUG"))                                                 \
                fprintf(stderr, "[b200-beagle] %s failed: %s (%s:%d)\n", #expr,              \
                        cudaGetErrorString(e__), __FILE__, __LINE__);                        \
            return e__ == cudaErrorMemoryAllocation ? BEAGLE_ERROR_OUT_OF_MEMORY             \
                                                    : BEAGLE_ERROR_GENERAL;                  \
        }                                                                                    \
    } while (0)

struct TimedScope {
    Instance* in;
    int cls;
    cudaEvent_t a = nullptr, b = nullptr;
    // `kernels`: how many kernel launches the bracket covers (a graph replay covers a whole plan)
    TimedScope(Instance* i, int c, int kernels = 1) : in(i), cls(c) {
        if (in->timing) {
            in->timedLaunches[cls] += kernels - 1;
            cudaEventCreate(&a);
            cudaEventCreate(&b);
            cudaEventRecord(a, in->stream);
        }
    }
    ~TimedScope() {
        if (in->timing) {
            cudaEventRecord(b, in->stream);
            in->timed[cls].push_back({a, b});
        }
    }
};

// reserve `bytes` in the pinned ring and copy `src` into it; nullptr if it cannot fit.  On wrap the stream is drained once,
// so a region is rewritten only after every launch that read it (by copy or in place) has finished.
static char* stageHost(Instance* in, const void* src, size_t bytes) {
    size_t need = (bytes + 255) & ~size_t(255);
    if (need > in->stageSize) return nullptr;
    if (in->stagePos + need > in->stageSize) {
        cudaStreamSynchronize(in->stream);
        in->stagePos = 0;
    }
    char* h = in->hStage + in->stagePos;
    memcpy(h, src, bytes);
    in->stagePos += need;
    return h;
}

// stage `src` and enqueue the H2D to the mirrored device ring; returns the device address
void* stage(Instance* in, const void* src, size_t bytes) {
    char* h = stageHost(in, src, bytes);
    if (h == nullptr) return nullptr;
    char* d = in->dStage + (h - in->hStage);
    if (cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, in->stream) != cudaSuccess) return nullptr;
    return d;
}

// stage `src` and return the device's view of the pinned bytes: the kernel reads them over PCIe, and no copy (with its
// wait between the copy engine and the kernel) sits in the stream before it
static const void* stageMapped(Instance* in, const void* src, size_t bytes) {
    char* h = stageHost(in, src, bytes);
    return h == nullptr ? nullptr : in->hStageDev + (h - in->hStage);
}

// small parameter upload straight into its device home (category rates, frequencies, ...)
int uploadSmall(Instance* in, void* dDst, const void* src, size_t bytes) {
    char* h = stageHost(in, src, bytes);
    if (h == nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(cudaMemcpyAsync(dDst, h, bytes, cudaMemcpyHostToDevice, in->stream));
    return BEAGLE_SUCCESS;
}

// partials live in ONE contiguous slab (index addressing in the walk kernels); a buffer index gets
// its slot on first use (tips that stay compact never consume one)
char* ensurePartials(Instance* in, int idx) {
    if (in->partials[idx] == nullptr) {
        if (in->nextSlot >= in->nSlots) return nullptr;
        in->slotOf[idx] = in->nextSlot++;
        in->partials[idx] = in->partialsBase + (size_t)in->slotOf[idx] * in->partialsElems * in->elemBytes();
    }
    return in->partials[idx];
}

bool validRange(int idx, int n) { return idx >= 0 && idx < n; }

void destroyInstance(Instance* in) {
    if (in->shard != nullptr) { shardedDestroy(in); delete in; return; }
    cudaSetDevice(in->device);
    exchangeRelease(in);
    if (in->stream) cudaStreamSynchronize(in->stream);
    cudaFree(in->partialsBase); cudaFree(in->states8Base); cudaFree(in->states32Base);
    for (CachedPlan& cp : in->planCache) { cp.dropGraph(); cudaFree(cp.dBlock); }
    cudaFree(in->dEigen); cudaFree(in->dMat); cudaFree(in->dEvec); cudaFree(in->dIncSums); cudaFree(in->dIncCounter);
    cudaFree(in->dRecipe);
    if (in->hMapped) cudaFreeHost(in->hMapped); cudaFree(in->dRates); cudaFree(in->dWeights);
    cudaFree(in->dFreqs); cudaFree(in->dScale); cudaFree(in->dPatternWeights);
    cudaFree(in->dPatternPartitions); cudaFree(in->dSite); cudaFree(in->dBlockSums); cudaFree(in->dOut);
    cudaFree(in->dCounter); cudaFree(in->dStage); cudaFree(in->dScratch);
    if (in->hStage) cudaFreeHost(in->hStage);
    if (in->hOut) cudaFreeHost(in->hOut);
    for (int c = 0; c < T_CLASSES; ++c)
        for (auto& ev : in->timed[c]) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
    if (in->stream) cudaStreamDestroy(in->stream);
    delete in;
}

// ---- resources ------------------------------------------------------------------------------
std::vector<BeagleResource> gResources;
std::vector<int> gShardDevices;          // devices of the pattern-sharded resource (empty: not offered)
int gShardResource = -1;                 // its resource number
std::vector<std::string> gResourceStrings;
BeagleResourceList gResourceList = {nullptr, 0};
std::once_flag gResourceOnce;

void buildResources() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
    gResourceStrings.reserve(2 * (n + 1));
    gResourceStrings.push_back("CPU (host)");
    gResourceStrings.push_back("no host implementation in this library | use a GPU resource (1..N)");
    for (int d = 0; d < n; ++d) {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, d) != cudaSuccess) { cudaGetLastError(); continue; }
        char buf[512];
        snprintf(buf, sizeof buf, "%s", prop.name);
        gResourceStrings.push_back(buf);
        snprintf(buf, sizeof buf, "Global memory (MB): %zu | SMs: %d | compute capability: %d.%d | "
                 "native walk kernels (sm_90a), fp64 arithmetic, fp64 or fp32 (4-state) partials",
                 (size_t)(prop.totalGlobalMem >> 20), prop.multiProcessorCount, prop.major, prop.minor);
        gResourceStrings.push_back(buf);
    }
    // the engine's own multi-GPU resource (multi.cu): one instance, site patterns sharded over the listed devices.
    // B200_SHARD_DEVICES="0,1,2,3" overrides the device list (a device may repeat: shards then share it -- test rigs).
    gShardDevices.clear();
    if (const char* env = getenv("B200_SHARD_DEVICES")) {
        for (const char* q = env; *q;) {
            char* end = nullptr;
            const long d = strtol(q, &end, 10);
            if (end == q) break;
            if (d >= 0 && d < n) gShardDevices.push_back((int)d);
            q = (*end == ',') ? end + 1 : end;
        }
    } else {
        for (int d = 0; d < n; ++d) gShardDevices.push_back(d);
    }
    if (gShardDevices.size() > (size_t)kMaxGroup) gShardDevices.resize(kMaxGroup);
    if (!gShardDevices.empty()) {
        char buf[512];
        snprintf(buf, sizeof buf, "GPU x %zu (pattern-sharded)", gShardDevices.size());
        gResourceStrings.push_back(buf);
        snprintf(buf, sizeof buf, "one instance over %zu GPUs | contiguous pattern blocks (Patterns.java:142-169 rule) | "
                 "per-shard sums added over NVLink inside the root kernel", gShardDevices.size());
        gResourceStrings.push_back(buf);
        gShardResource = (int)(gResourceStrings.size() / 2) - 1;
    }
    size_t count = gResourceStrings.size() / 2;
    gResources.resize(count);
    for (size_t r = 0; r < count; ++r) {
        gResources[r].name = const_cast<char*>(gResourceStrings[2 * r].c_str());
        gResources[r].description = const_cast<char*>(gResourceStrings[2 * r + 1].c_str());
        gResources[r].supportFlags = (r == 0) ? (BEAGLE_FLAG_PROCESSOR_CPU | BEAGLE_FLAG_FRAMEWORK_CPU) : kSupportedFlags;
        gResources[r].requiredFlags = (r == 0) ? BEAGLE_FLAG_FRAMEWORK_CPU : BEAGLE_FLAG_FRAMEWORK_CUDA;
    }
    gResourceList.list = gResources.data();
    gResourceList.length = (int)count;
}

char gImplName[] = "B200-CUDA-Double";
char gImplNameSingle[] = "B200-CUDA-Single";     // fp32 partials storage, fp64 arithmetic
char gImplDesc[] = "sm_90a walk kernels: one launch per operation list, shared-memory operand stack";

// ---- op planning ------------------------------------------------------------------------------

// Execution plan of one operation list.
//
// Pattern columns never interact, so ANY topological order of the list is valid, and independent
// subtrees of the list may run concurrently.  The plan cuts the op forest into PHASES of disjoint
// subtrees of at most T ops ("all maximal subtrees with <= T ops", then recurse on what is left):
//   * every (subtree, pattern tile) pair is one independent walk -> grid.y = subtrees of the phase,
//     which multiplies the warps in flight (latency hiding) and shortens the dependent chain from
//     n ops to ~phases*T;
//   * inside a subtree ops run in Sethi-Ullman order (deeper-need child first), which minimises the
//     number of live intermediate results = operand-stack slots;
//   * results crossing a phase boundary go through global memory (L2), everything else through the
//     shared-memory stack.
// Lists with hazards the forest model does not cover (a buffer written twice, read-before-write,
// a result consumed by two ops) run as ONE subtree in the caller's order.
struct Sub { int begin, end, pBase, pLimit; };     // op positions [begin,end) applied to patterns [pBase,pLimit)
struct Plan {
    std::vector<int> order;          // execution position -> index into the caller's list
    std::vector<Sub> subs;           // position ranges, grouped by phase
    std::vector<int> phaseStart;     // index into subs; size = phases + 1
};

void planPhases(const std::vector<HostOp>& ops, int nBuffers, bool allowReorder, int fixedT, int wantSubs, int minT,
                int smallRemainder, Plan& plan) {
    const int n = (int)ops.size();
    auto single = [&]() {
        plan.order.resize(n);
        for (int k = 0; k < n; ++k) plan.order[k] = k;
        plan.subs.assign(1, Sub{0, n, 0, 0});
        plan.phaseStart = {0, 1};
    };
    if (!allowReorder || n < 2) { single(); return; }
    std::vector<int> writer(nBuffers, -1);
    for (int k = 0; k < n; ++k) {
        if (writer[ops[k].dest] >= 0) { single(); return; }
        writer[ops[k].dest] = k;
    }
    std::vector<int> ch0(n, -1), ch1(n, -1), parent(n, -1);
    for (int k = 0; k < n; ++k) {
        const int a = writer[ops[k].c1], b = writer[ops[k].c2];
        if (a >= 0) { if (a >= k || parent[a] >= 0) { single(); return; } ch0[k] = a; parent[a] = k; }
        if (b >= 0 && ops[k].c2 != ops[k].c1) { if (b >= k || parent[b] >= 0) { single(); return; } ch1[k] = b; parent[b] = k; }
        if (ops[k].dest == ops[k].c1 || ops[k].dest == ops[k].c2) { single(); return; }
    }
    std::vector<char> alive(n, 1);
    std::vector<int> size(n), need(n);
    std::vector<std::pair<int, int>> stack;
    plan.order.clear(); plan.order.reserve(n);
    plan.subs.clear(); plan.phaseStart.assign(1, 0);
    int remaining = n;
    while (remaining > 0) {
        // per-phase subtree bound: enough subtrees to fill the machine, re-evaluated on what is left
        // (a remainder of a couple of dozen ops is cheaper as one launch than as several tiny phases)
        const int T = fixedT > 0 ? fixedT : (remaining <= smallRemainder ? remaining : std::max(minT, (remaining + wantSubs - 1) / wantSubs));
        for (int k = 0; k < n; ++k) {
            if (!alive[k]) continue;
            const int a = (ch0[k] >= 0 && alive[ch0[k]]) ? ch0[k] : -1;
            const int b = (ch1[k] >= 0 && alive[ch1[k]]) ? ch1[k] : -1;
            size[k] = 1 + (a >= 0 ? size[a] : 0) + (b >= 0 ? size[b] : 0);
            int na = a >= 0 ? need[a] : 0, nb = b >= 0 ? need[b] : 0;
            if (na < nb) std::swap(na, nb);
            need[k] = std::max(1, std::max(na, nb + (nb > 0 ? 1 : 0)));
        }
        for (int r = 0; r < n; ++r) {
            if (!alive[r] || size[r] > T) continue;
            if (parent[r] >= 0 && size[parent[r]] <= T) continue;       // not maximal
            const int begin = (int)plan.order.size();
            stack.push_back({r, 0});
            while (!stack.empty()) {
                auto [k, stageNo] = stack.back();
                stack.pop_back();
                if (stageNo == 1) { plan.order.push_back(k); continue; }
                stack.push_back({k, 1});
                const int a = (ch0[k] >= 0 && alive[ch0[k]]) ? ch0[k] : -1;
                const int b = (ch1[k] >= 0 && alive[ch1[k]]) ? ch1[k] : -1;
                const int na = a >= 0 ? need[a] : -1, nb = b >= 0 ? need[b] : -1;
                // the child pushed LAST is visited FIRST: visit the larger need first
                if (na >= nb) { if (b >= 0) stack.push_back({b, 0}); if (a >= 0) stack.push_back({a, 0}); }
                else          { if (a >= 0) stack.push_back({a, 0}); if (b >= 0) stack.push_back({b, 0}); }
            }
            plan.subs.push_back(Sub{begin, (int)plan.order.size(), 0, 0});
        }
        // retire this phase's ops only now, so that maximality was judged on a consistent snapshot
        for (int q = plan.subs[plan.phaseStart.back()].begin; q < (int)plan.order.size(); ++q) alive[plan.order[q]] = 0;
        // longest subtrees first: blocks are dispatched in grid order, so the long walks start early
        std::stable_sort(plan.subs.begin() + plan.phaseStart.back(), plan.subs.end(),
                         [](const Sub& a, const Sub& b) { return (a.end - a.begin) > (b.end - b.begin); });
        remaining = n - (int)plan.order.size();
        plan.phaseStart.push_back((int)plan.subs.size());
    }
}

// Pre-order lists form an OUT-forest (pre[node] needs pre[parent]); ops of equal depth are independent.
// One launch per depth level, every op its own walk (grid.y = ops of the level).
void planLevels(const std::vector<HostOp>& ops, int nBuffers, Plan& plan) {
    const int n = (int)ops.size();
    std::vector<int> writer(nBuffers, -1), level(n, 0);
    bool hazard = false;
    for (int k = 0; k < n; ++k) { if (writer[ops[k].dest] >= 0) hazard = true; writer[ops[k].dest] = k; }
    int maxLevel = 0;
    for (int k = 0; k < n && !hazard; ++k) {
        for (int src : {ops[k].c1, ops[k].c2}) {
            const int w = writer[src];
            if (w < 0) continue;
            if (w >= k) { hazard = true; break; }
            level[k] = std::max(level[k], level[w] + 1);
        }
        maxLevel = std::max(maxLevel, level[k]);
    }
    plan.order.resize(n);
    for (int k = 0; k < n; ++k) plan.order[k] = k;
    plan.subs.clear();
    if (hazard) { plan.subs.assign(1, Sub{0, n, 0, 0}); plan.phaseStart = {0, 1}; return; }
    std::stable_sort(plan.order.begin(), plan.order.end(), [&](int a, int b) { return level[a] < level[b]; });
    plan.phaseStart.assign(1, 0);
    for (int pos = 0; pos < n; ++pos) {
        if (pos > 0 && level[plan.order[pos]] != level[plan.order[pos - 1]]) plan.phaseStart.push_back((int)plan.subs.size());
        plan.subs.push_back(Sub{pos, pos + 1, 0, 0});
    }
    plan.phaseStart.push_back((int)plan.subs.size());
}

// Pre-order lists, the mirror image of planPhases: op(node) needs op(parent) (its c1 is the parent's destination) and
// nothing else from this list, so the ops form an OUT-forest.  Subtrees of that forest are cut bottom-up exactly like the
// post-order plan ("all maximal subtrees with <= T ops", then again on what is left) and the phases run in REVERSE order
// of extraction: the crown first, the many independent subtrees last.  Inside a subtree ops run in depth-first pre-order,
// so the op after a node is its first child and finds pre[parent] in the walking thread's registers.
// Anything the forest model does not cover (double write, read-before-write, a c2 produced in this list) -> planLevels.
void planPreorderPhases(const std::vector<HostOp>& ops, int nBuffers, int fixedT, int wantSubs, int minT,
                        int smallRemainder, Plan& plan) {
    const int n = (int)ops.size();
    std::vector<int> writer(nBuffers, -1), parent(n, -1);
    bool ok = n >= 2;
    for (int k = 0; k < n && ok; ++k) { ok = writer[ops[k].dest] < 0; writer[ops[k].dest] = k; }
    for (int k = 0; k < n && ok; ++k) {
        const int a = writer[ops[k].c1];
        ok = writer[ops[k].c2] < 0 && (a < 0 || a < k) && ops[k].dest != ops[k].c1 && ops[k].dest != ops[k].c2;
        parent[k] = a;
    }
    if (!ok) { planLevels(ops, nBuffers, plan); return; }
    std::vector<std::vector<int>> kids(n);
    for (int k = 0; k < n; ++k) if (parent[k] >= 0) kids[parent[k]].push_back(k);
    std::vector<char> alive(n, 1);
    std::vector<int> size(n), stack;
    std::vector<std::vector<int>> phases;          // roots of the subtrees of each extracted phase
    int remaining = n;
    while (remaining > 0) {
        const int T = fixedT > 0 ? fixedT : (remaining <= smallRemainder ? remaining : std::max(minT, (remaining + wantSubs - 1) / wantSubs));
        for (int k = n - 1; k >= 0; --k) {          // children have larger indices than their parent
            if (!alive[k]) continue;
            size[k] = 1;
            for (int c : kids[k]) if (alive[c]) size[k] += size[c];
        }
        std::vector<int> roots;
        for (int r = 0; r < n; ++r)
            if (alive[r] && size[r] <= T && !(parent[r] >= 0 && alive[parent[r]] && size[parent[r]] <= T)) roots.push_back(r);
        for (int r : roots) {                       // retire after the snapshot was judged
            stack.assign(1, r);
            while (!stack.empty()) {
                const int k = stack.back(); stack.pop_back();
                if (!alive[k]) continue;
                alive[k] = 0; --remaining;
                for (int c : kids[k]) if (alive[c]) stack.push_back(c);
            }
        }
        phases.push_back(std::move(roots));
    }
    // emit: last extracted phase first; membership of a subtree = the ops retired with its root
    std::vector<int> phaseOf(n, -1), rootOf(n, -1);
    for (int ph = 0; ph < (int)phases.size(); ++ph)
        for (int r : phases[ph]) { phaseOf[r] = ph; rootOf[r] = r; }
    for (int k = 0; k < n; ++k)                      // parents precede children: inherit unless k is itself a root
        if (rootOf[k] < 0) { rootOf[k] = rootOf[parent[k]]; phaseOf[k] = phaseOf[parent[k]]; }
    plan.order.clear(); plan.order.reserve(n);
    plan.subs.clear(); plan.phaseStart.assign(1, 0);
    for (int ph = (int)phases.size() - 1; ph >= 0; --ph) {
        for (int r : phases[ph]) {
            const int begin = (int)plan.order.size();
            stack.assign(1, r);
            while (!stack.empty()) {                 // depth-first pre-order restricted to this subtree
                const int k = stack.back(); stack.pop_back();
                plan.order.push_back(k);
                for (int q = (int)kids[k].size() - 1; q >= 0; --q)
                    if (rootOf[kids[k][q]] == r) stack.push_back(kids[k][q]);
            }
            plan.subs.push_back(Sub{begin, (int)plan.order.size(), 0, 0});
        }
        std::stable_sort(plan.subs.begin() + plan.phaseStart.back(), plan.subs.end(),
                         [](const Sub& a, const Sub& b) { return (a.end - a.begin) > (b.end - b.begin); });
        plan.phaseStart.push_back((int)plan.subs.size());
    }
}

// register forwarding: inside one subtree walk a thread re-reads, as a child, exactly the cell it wrote for the previous
// op -- flag it (bit 1), with that child moved to position 1 (the product commutes exactly); tip: the op's virtual tips
void forwardFromPrevious(Op4& d, const Op4& pv, bool preOrder, int4* tip) {
    if (pv.pBegin != d.pBegin || pv.pEnd != d.pEnd) return;
    const bool v1 = (d.pad_ & 4) != 0, v2 = (d.pad_ & 8) != 0;
    if (d.c1 >= 0 && !v1 && d.c1 == pv.dest) d.pad_ |= 2;     // pre-order: pre[parent] is the previous result
    else if (!preOrder && d.c2 >= 0 && !v2 && d.c2 == pv.dest) {
        std::swap(d.c1, d.c2); std::swap(d.m1, d.m2);
        if (tip) *tip = make_int4(tip->z, tip->w, tip->x, tip->y);
        d.pad_ = (d.pad_ & ~12) | (v1 ? 8 : 0) | 2;
    }
}

// ---- sibling stack of the staged eigen walk (k_walk4p, walk4e.cu) -----------------------------------------------------
// Inside one (subtree, pattern tile) walk a result is taken by the next op from registers, or read back later as the
// sibling of some op, or read by another walk only.  Results of the second kind also go to a per-warp shared-memory slot:
// the lowest free one when the result is written, freed at its last read that does not come from registers.  With all
// `depth` slots taken the value travels through memory as before.  Forwarded, tip, virtual and cross-phase children never
// take a slot.  Every result is still stored to global memory (other walks, later lists, the root and getPartials read it
// there), so a kernel that ignores the slot bytes computes the same thing.  Needs the final forwarding flags.
// subDepth[s]: slots the walk of subtree s uses; fromStack / fromMemory: internal children read from a slot / from memory.
void assignStackSlots(std::vector<Op4>& ops, const std::vector<Sub>& subs, int depth, std::vector<int>& subDepth,
                      long& fromStack, long& fromMemory) {
    // the partials slot child ch is read from in memory, or -1 (tip, virtual cherry, forwarded in registers)
    auto memoryChild = [](const Op4& d, int ch) -> int {
        const int c = ch == 0 ? d.c1 : d.c2;
        if (c < 0 || (d.pad_ & (4 << ch)) || (ch == 0 && (d.pad_ & 2))) return -1;
        return c;
    };
    int keys = 1;
    for (const Op4& d : ops) keys = std::max(keys, 1 + std::max(d.dest, std::max(d.c1, d.c2)));
    std::vector<int> lastRead(keys, -1), slotOf(keys, -1), freeAt(keys, -1), lastReadOf(ops.size(), -1);
    subDepth.assign(subs.size(), 0);
    for (size_t s = 0; s < subs.size(); ++s) {
        const int b = subs[s].begin, e = subs[s].end;
        for (int pos = e - 1; pos >= b; --pos) {                  // last memory read of each result before its rewrite
            const Op4& d = ops[pos];
            lastReadOf[pos] = lastRead[d.dest];
            lastRead[d.dest] = -1;
            for (int ch = 0; ch < 2; ++ch) {
                const int c = memoryChild(d, ch);
                if (c >= 0 && lastRead[c] < 0) lastRead[c] = pos;
            }
        }
        unsigned freeMask = (1u << depth) - 1u;
        for (int pos = b; pos < e; ++pos) {
            Op4& d = ops[pos];
            int src[2] = {0xFF, 0xFF};
            for (int ch = 0; ch < 2; ++ch) {
                const int c = memoryChild(d, ch);
                if (c < 0) continue;
                if (slotOf[c] >= 0) { src[ch] = slotOf[c]; ++fromStack; } else ++fromMemory;
            }
            for (int ch = 0; ch < 2; ++ch) {
                const int c = memoryChild(d, ch);
                if (c >= 0 && slotOf[c] >= 0 && freeAt[c] == pos) { freeMask |= 1u << slotOf[c]; slotOf[c] = -1; }
            }
            if (slotOf[d.dest] >= 0) { freeMask |= 1u << slotOf[d.dest]; slotOf[d.dest] = -1; }     // stale value
            int dst = 0xFF;
            if (lastReadOf[pos] > pos && freeMask != 0) {
                dst = __builtin_ctz(freeMask);
                freeMask &= ~(1u << dst);
                slotOf[d.dest] = dst;
                freeAt[d.dest] = lastReadOf[pos];
                subDepth[s] = std::max(subDepth[s], dst + 1);
            }
            d.slots = (unsigned)src[0] | ((unsigned)src[1] << 8) | ((unsigned)dst << 16);
        }
        for (int pos = b; pos < e; ++pos) {                       // leave no marks for the next subtree
            const Op4& d = ops[pos];
            lastRead[d.dest] = slotOf[d.dest] = -1;
            for (int ch = 0; ch < 2; ++ch) if (memoryChild(d, ch) >= 0) lastRead[memoryChild(d, ch)] = -1;
        }
    }
}

// launch the phases of a prepared plan (device-resident op records + subtree table)
// eigenSlot >= 0: the 4-state list runs in eigen form (walk4e.cu) with that slot's V / V^-1; aligned: no pattern windows;
// nSnap: virtual cherries the list produces (their recipes are snapshot first); virt: the records name virtual cherries;
// phaseSlots: sibling-stack depth of each phase (eigen-form walks)
cudaError_t launchPlan(Instance* in, const void* dOps, const void* dSubs, const std::vector<int>& phaseStart,
                       const std::vector<int>& phaseDepth, const std::vector<int>& phaseSlots, bool fourPath, int maxWindow,
                       bool preOrder, int eigenSlot = -1,
                       bool aligned = false, const void* dSnap = nullptr, int nSnap = 0, const void* dVirtTips = nullptr) {
    const bool virt = dVirtTips != nullptr;
    cudaError_t e = cudaSuccess;
    if (nSnap > 0) {
        TimedScope ts(in, T_PARTIALS);
        e = launchCherrySnapshot(in, static_cast<const int4*>(dSnap), nSnap);
    }
    for (size_t ph = 0; ph + 1 < phaseStart.size() && e == cudaSuccess; ++ph) {
        const int s0 = phaseStart[ph], s1 = phaseStart[ph + 1];
        if (s1 <= s0) continue;
        TimedScope ts(in, T_PARTIALS);
        if (fourPath && eigenSlot >= 0 && !preOrder && (ph >= phaseDepth.size() || phaseDepth[ph] == 0)) {
            e = launchWalk4E(in, static_cast<const Op4*>(dOps), static_cast<const int4*>(dSubs) + s0, s1 - s0, maxWindow,
                             aligned, in->hEigen.data() + (size_t)eigenSlot * 36, static_cast<const int4*>(dVirtTips),
                             ph < phaseSlots.size() ? phaseSlots[ph] : 0);
            continue;
        }
        if (virt) return cudaErrorInvalidValue;          // no other walk reads virtual cherries
        e = fourPath ? launchWalk4(in, static_cast<const Op4*>(dOps), static_cast<const int4*>(dSubs) + s0, s1 - s0,
                                   ph < phaseDepth.size() ? phaseDepth[ph] : 0, maxWindow, preOrder)
                     : launchWalkGeneric(in, static_cast<const DevOp*>(dOps), static_cast<const int4*>(dSubs) + s0, s1 - s0,
                                         maxWindow, preOrder);
    }
    return e;
}

// cum[p] += sum_k log factor_k[p] for the in-list cumulative groups of a plan (after its phases, same stream)
cudaError_t accumulateInList(Instance* in, const std::vector<CumGroup>& groups) {
    for (const CumGroup& g : groups) {
        int* dIdx = static_cast<int*>(stage(in, g.indices.data(), sizeof(int) * g.indices.size()));
        if (dIdx == nullptr) return cudaErrorMemoryAllocation;
        cudaError_t e = launchScaleAccumulate(in, dIdx, (int)g.indices.size(), in->dScale + (size_t)g.cum * in->Ppad, 1.0,
                                              g.pBegin, g.pEnd);
        if (e != cudaSuccess) return e;
        in->scaleIsLog[g.cum] = 1;
    }
    return cudaSuccess;
}

// per-node scale buffers written by a list hold raw factors (logs under SCALERS_LOG)
void noteScaleWrites(Instance* in, const std::vector<HostOp>& hops) {
    for (const HostOp& o : hops) if (o.sw >= 0) in->scaleIsLog[o.sw] = in->logScalers ? 1 : 0;
}

// ---- virtual cherries (walk4e.cu) ----------------------------------------------------------------------------------
// A tip x tip op without rescaling in a list the eigen-form walk runs on k_walk4p is not run: its consumers recompute
// colA ⊙ colB from a recipe (the two P blocks, snapshot when the list runs) and the two tips' state bytes.  Its partials
// are written only when something else reads the buffer, through storeCherries -- the one place that happens.

// every reader of stored partials other than k_walk4pv calls this with the buffers it is about to read: virtual cherries
// among them get their partials written (they stay virtual-readable: the recipe is still valid)
cudaError_t storeCherries(Instance* in, const int* bufs, int count) {
    if (in->cherryTip1.empty()) return cudaSuccess;
    std::vector<int4> items;
    for (int k = 0; k < count; ++k) {
        const int b = bufs[k];
        if (!validRange(b, in->nBuffers) || in->cherryTip1[b] < 0 || in->cherryStored[b]) continue;
        items.push_back(make_int4(in->slotOf[b], b, in->cherryTip1[b], in->cherryTip2[b]));
        in->cherryStored[b] = 1;
    }
    if (items.empty()) return cudaSuccess;
    const int4* dItems = static_cast<const int4*>(stage(in, items.data(), sizeof(int4) * items.size()));
    cudaError_t e = cudaErrorMemoryAllocation;
    if (dItems != nullptr) {
        TimedScope ts(in, T_PARTIALS);
        e = launchCherryStore(in, dItems, (int)items.size());
    }
    if (e != cudaSuccess) for (const int4& it : items) in->cherryStored[it.y] = 0;
    return e;
}

// children a list reads from outside itself as stored partials
cudaError_t storeExternal(Instance* in, const std::vector<CherryRef>& external) {
    std::vector<int> bufs;
    for (const CherryRef& x : external) if (x.tip1 < 0) bufs.push_back(x.buf);
    return storeCherries(in, bufs.data(), (int)bufs.size());
}

// tip t is about to change: the cherries computed from it get their partials written and are plain partials from now on
cudaError_t settleCherriesOf(Instance* in, int t) {
    std::vector<int> deps;
    for (int b = 0; b < (int)in->cherryTip1.size(); ++b)
        if (in->cherryTip1[b] >= 0 && (in->cherryTip1[b] == t || in->cherryTip2[b] == t)) deps.push_back(b);
    const cudaError_t e = storeCherries(in, deps.data(), (int)deps.size());
    if (e == cudaSuccess) for (int b : deps) in->cherryTip1[b] = -1;
    return e;
}

// a list ran: its destinations hold real partials, except the virtual cherries it produced
void noteCherryWrites(Instance* in, const std::vector<HostOp>& hops, const std::vector<CherryRef>& cherries) {
    if (in->cherryTip1.empty()) return;
    for (const HostOp& o : hops) in->cherryTip1[o.dest] = -1;
    for (const CherryRef& c : cherries) {
        in->cherryTip1[c.buf] = c.tip1; in->cherryTip2[c.buf] = c.tip2; in->cherryStored[c.buf] = 0;
    }
}

// validation (no side effects) of an operation list, then lazy allocation / kind changes of its destinations
int prepareOps(Instance* in, const std::vector<HostOp>& hops, bool byPartition) {
    for (const HostOp& o : hops) {
        if (!validRange(o.dest, in->nBuffers) || !validRange(o.c1, in->nBuffers) ||
            !validRange(o.c2, in->nBuffers) || !validRange(o.m1, in->nMatrices) ||
            !validRange(o.m2, in->nMatrices))
            return BEAGLE_ERROR_OUT_OF_RANGE;
        if (o.sw != BEAGLE_OP_NONE && !validRange(o.sw, in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
        if (o.sr != BEAGLE_OP_NONE && !validRange(o.sr, in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
        if (o.cum != BEAGLE_OP_NONE && !validRange(o.cum, in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
        if (byPartition && !validRange(o.part, in->partitionCount)) return BEAGLE_ERROR_OUT_OF_RANGE;
    }
    {
        // a child must hold data: compact states, partials, or the destination of an op of this very list
        std::vector<char> written(in->nBuffers, 0);
        for (const HostOp& o : hops) written[o.dest] = 1;
        auto holdsData = [&](int b) { return written[b] || in->partials[b] != nullptr || in->states32[b] != nullptr; };
        for (const HostOp& o : hops) {
            if (!holdsData(o.c1) || !holdsData(o.c2)) return BEAGLE_ERROR_OUT_OF_RANGE;
            // pre-order: c1 is pre[parent], a partials buffer by construction
            if (o.kind == 1 && !written[o.c1] && in->states32[o.c1] != nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
        }
    }
    for (const HostOp& o : hops) {
        if (ensurePartials(in, o.dest) == nullptr) return BEAGLE_ERROR_OUT_OF_MEMORY;
        if (in->states32[o.dest] != nullptr) in->bufferEpoch++;
        in->states8[o.dest] = nullptr;      // a written buffer holds partials from now on
        in->states32[o.dest] = nullptr;
    }
    return BEAGLE_SUCCESS;
}

// The eigen-form walk serves a post-order 4-state list when every matrix it names was computed by
// updateTransitionMatrices from the CURRENT content of ONE real eigen slot; returns that slot or -1.
int eigenFormSlot(const Instance* in, const std::vector<HostOp>& hops) {
    if (!in->eigenWalk || in->matCP == 0 || in->walkVariant != 0 || hops.empty() || hops[0].kind == 1) return -1;
    const int E = in->matEigen[hops[0].m1];
    if (E < 0 || !in->eigenReal[E]) return -1;
    const unsigned gen = in->eigenGen[E];
    for (const HostOp& o : hops)
        if (in->matEigen[o.m1] != E || in->matEigen[o.m2] != E || in->matEigenGen[o.m1] != gen || in->matEigenGen[o.m2] != gen)
            return -1;
    return E;
}

int planAndLaunch(Instance* in, const std::vector<HostOp>& hops, bool byPartition) {
    const int n = (int)hops.size();
    if (n == 0) return BEAGLE_SUCCESS;
    // ---- plan cache: MCMC re-issues identical lists all the time (every move that keeps the topology and
    // dirties all nodes, in BEAST's two buffer-index parities); a hit skips validation, planning and the H2D copy.
    static_assert(sizeof(HostOp) == 10 * sizeof(int), "HostOp is compared bytewise");
    if (in->planCacheSize > 0) {
        for (CachedPlan& cp : in->planCache) {
            if (cp.dBlock == nullptr || cp.n != n || cp.byPartition != byPartition || cp.epoch != in->bufferEpoch ||
                memcmp(cp.key.data(), hops.data(), sizeof(HostOp) * (size_t)n) != 0)
                continue;
            const int eigenSlot = cp.fourPath ? eigenFormSlot(in, hops) : -1;
            // records that name virtual cherries need the eigen form, and an outside child read as a cherry must still be it
            bool stale = cp.readsVirtual && eigenSlot < 0;
            for (const CherryRef& x : cp.external)
                stale = stale || (x.tip1 >= 0 && (in->cherryTip1[x.buf] != x.tip1 || in->cherryTip2[x.buf] != x.tip2));
            if (stale) { cp.dropGraph(); cp.n = -1; continue; }
            CUDA_OK(storeExternal(in, cp.external));
            cp.lastUse = ++in->planClock;
            cp.hits++;
            const unsigned eigenGenNow = eigenSlot >= 0 ? in->eigenGen[eigenSlot] : 0u;
            const void* dSnap = static_cast<char*>(cp.dBlock) + cp.snapOffset;
            const int nSnap = (int)cp.cherries.size();
            const void* dTips = cp.readsVirtual ? static_cast<char*>(cp.dBlock) + cp.tipsOffset : nullptr;
            // a captured graph carries the kernel choice and V / V^-1 by value: stale once the eigen system moved on
            if (cp.graphExec != nullptr && (cp.graphEigen != eigenSlot || cp.graphEigenGen != eigenGenNow)) {
                // same kernels, new V / V^-1 (a substitution-model move): patch the captured launches in place
                if (cp.graphAllEigen && eigenSlot >= 0 && cp.graphEigen == eigenSlot &&
                    updateWalk4EGraph(cp.graphExec, cp.graphKernelNodes, in->hEigen.data() + (size_t)eigenSlot * 36) == cudaSuccess) {
                    cp.graphEigenGen = eigenGenNow;
                } else {
                    cudaGetLastError();
                    cp.dropGraph();
                    cp.hits = 1;
                    if (++cp.graphInvalidations >= 4) cp.graphFailed = true;     // the kernel choice flips every step: plain launches
                }
            }
            // A plan that keeps coming back and needs several dependent launches is replayed as ONE graph launch:
            // on small alignments the host-side launch cost, not the kernels, sets the pace.
            int launches = nSnap > 0;
            for (size_t ph = 0; ph + 1 < cp.phaseStart.size(); ++ph) launches += cp.phaseStart[ph + 1] > cp.phaseStart[ph];
            // (in-list cumulative scaling stages its index lists per call: those plans keep the plain launches)
            if (in->useGraphs && launches >= 2 && cp.cumGroups.empty()) {
                if (cp.graphExec == nullptr && !cp.graphFailed && cp.hits >= 2 && !in->timing &&
                    cudaStreamBeginCapture(in->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
                    const cudaError_t e1 = launchPlan(in, cp.dBlock, static_cast<char*>(cp.dBlock) + cp.subsOffset, cp.phaseStart,
                                                      cp.phaseDepth, cp.phaseSlots, cp.fourPath, cp.maxWindow, cp.preOrder, eigenSlot,
                                                      !cp.byPartition, dSnap, nSnap, dTips);
                    cp.graphEigen = eigenSlot;
                    cp.graphEigenGen = eigenGenNow;
                    cudaGraph_t g = nullptr;
                    const cudaError_t e2 = cudaStreamEndCapture(in->stream, &g);
                    if (e1 != cudaSuccess || e2 != cudaSuccess || g == nullptr ||
                        cudaGraphInstantiate(&cp.graphExec, g, 0) != cudaSuccess) {
                        cp.graphExec = nullptr;
                        cp.graphFailed = true;
                        if (g) cudaGraphDestroy(g);
                    } else {
                        cp.graph = g;
                        cp.graphKernelNodes.clear();
                        cp.graphAllEigen = cp.fourPath && eigenSlot >= 0 && !cp.preOrder;
                        for (int dpt : cp.phaseDepth) cp.graphAllEigen = cp.graphAllEigen && dpt == 0;
                        size_t nn = 0;
                        if (cudaGraphGetNodes(g, nullptr, &nn) == cudaSuccess && nn > 0) {
                            std::vector<cudaGraphNode_t> nodes(nn);
                            cudaGraphNodeType ty;
                            if (cudaGraphGetNodes(g, nodes.data(), &nn) == cudaSuccess)
                                for (size_t q = 0; q < nn; ++q)
                                    if (cudaGraphNodeGetType(nodes[q], &ty) == cudaSuccess && ty == cudaGraphNodeTypeKernel)
                                        cp.graphKernelNodes.push_back(nodes[q]);
                        }
                        if (cp.graphKernelNodes.empty()) cp.graphAllEigen = false;
                    }
                    if (getenv("B200_BEAGLE_DEBUG"))
                        fprintf(stderr, "[b200-beagle] graph %s: %d launches\n", cp.graphExec ? "captured" : "capture failed",
                                launches);
                    cudaGetLastError();
                }
                if (cp.graphExec != nullptr) {
                    TimedScope ts(in, T_PARTIALS, launches);
                    CUDA_OK(cudaGraphLaunch(cp.graphExec, in->stream));
                    noteScaleWrites(in, hops);
                    noteCherryWrites(in, hops, cp.cherries);
                    return BEAGLE_SUCCESS;
                }
            }
            CUDA_OK(launchPlan(in, cp.dBlock, static_cast<char*>(cp.dBlock) + cp.subsOffset, cp.phaseStart, cp.phaseDepth,
                               cp.phaseSlots, cp.fourPath, cp.maxWindow, cp.preOrder, eigenSlot, !cp.byPartition, dSnap, nSnap,
                               dTips));
            CUDA_OK(accumulateInList(in, cp.cumGroups));
            noteScaleWrites(in, hops);
            noteCherryWrites(in, hops, cp.cherries);
            return BEAGLE_SUCCESS;
        }
    }
    {
        const int rcPrepare = prepareOps(in, hops, byPartition);
        if (rcPrepare != BEAGLE_SUCCESS) return rcPrepare;
    }
    const bool fourState = in->matCP > 0;
    const bool preOrder = hops[0].kind == 1;
    const int eigenSlot = fourState ? eigenFormSlot(in, hops) : -1;
    std::vector<char> written(in->nBuffers, 0);
    std::vector<int> firstWrite(in->nBuffers, n);
    for (int k = n - 1; k >= 0; --k) { written[hops[k].dest] = 1; firstWrite[hops[k].dest] = k; }
    // ---- virtual cherries: the ops that are not run (each tip x tip op without rescaling whose destination this list
    // writes once and reads only afterwards), and whether any op record names a virtual child
    std::vector<CherryRef> cherries;
    std::vector<int4> snap;
    std::vector<HostOp> kept;
    bool readsVirtual = false;
    if (!in->cherryTip1.empty() && !byPartition && !preOrder && eigenSlot >= 0 && !in->stackTail) {
        std::vector<int> writes(in->nBuffers, 0), firstRead(in->nBuffers, n);
        for (int k = 0; k < n; ++k) {
            writes[hops[k].dest]++;
            firstRead[hops[k].c1] = std::min(firstRead[hops[k].c1], k);
            firstRead[hops[k].c2] = std::min(firstRead[hops[k].c2], k);
        }
        for (int k = 0; k < n; ++k) {
            const HostOp& o = hops[k];
            if (in->states8[o.c1] != nullptr && in->states8[o.c2] != nullptr && o.sw == BEAGLE_OP_NONE &&
                o.sr == BEAGLE_OP_NONE && o.cum == BEAGLE_OP_NONE && writes[o.dest] == 1 && firstRead[o.dest] > k) {
                cherries.push_back(CherryRef{o.dest, o.c1, o.c2});
                snap.push_back(make_int4(o.dest, o.m1, o.m2, 0));
            } else {
                kept.push_back(o);
            }
        }
        if (kept.empty()) { cherries.clear(); snap.clear(); }       // nothing would run: keep the list as it is
        readsVirtual = !cherries.empty();
        for (const HostOp& o : hops)
            for (int c : {o.c1, o.c2})
                readsVirtual = readsVirtual || (!written[c] && in->states32[c] == nullptr && in->cherryTip1[c] >= 0);
    }
    Plan plan;
    int maxWindow = in->Ppad;
    // patterns one warp owns: FMA kernel (32/CP)*R, tensor kernels 8*R resp. 16
    const int patsPerWarp = !fourState ? 16 : (in->walkVariant == 2 ? 8 * in->tensorR : (32 / in->matCP) * in->walkR);
    const int warpsPerSM = fourState ? 32 : 12;      // resident warps the kernel family can hold per SM
    auto wantSubsFor = [&](int window) {
        const int warpsPerSub = std::max(1, (window + patsPerWarp - 1) / patsPerWarp);
        // enough (subtree x tile) walks to fill every SM, oversubscribed for balance
        // oversubscription for balance: 2x where a subtree is only a few warps wide (small alignments), 1x where every
        // subtree already spreads over dozens of warps -- longer walks forward more results through registers
        // (measured: cfg 2 +3 %, codon +5 %, benchmark2 +4 %; benchmark1-sized inputs -1..-3 % if forced to 1)
        const int over = in->phaseOversub > 0 ? in->phaseOversub : (warpsPerSub >= 32 ? 1 : 2);
        return std::max(1, over * ((in->smCount * warpsPerSM + warpsPerSub - 1) / warpsPerSub));
    };
    if (!byPartition && !preOrder) {
        planPhases(cherries.empty() ? hops : kept, in->nBuffers, in->reorder != 0, in->phaseT, wantSubsFor(in->Ppad),
                   in->phaseTmin, in->phaseSmall, plan);
        // only k_walk4p reads virtual children: if some phase of this plan would run elsewhere, every op runs as usual
        bool served = true;
        for (size_t ph = 0; readsVirtual && ph + 1 < plan.phaseStart.size(); ++ph) {
            const int nSubs = plan.phaseStart[ph + 1] - plan.phaseStart[ph];
            served = served && (nSubs == 0 || walk4pServes(in, nSubs, in->Ppad));
        }
        if (!served) {
            readsVirtual = false;
            if (!cherries.empty()) {
                cherries.clear(); snap.clear(); kept.clear();
                planPhases(hops, in->nBuffers, in->reorder != 0, in->phaseT, wantSubsFor(in->Ppad), in->phaseTmin,
                           in->phaseSmall, plan);
            }
        }
        for (Sub& sb : plan.subs) { sb.pBase = 0; sb.pLimit = in->Ppad; }
    }
    // the ops that run
    const std::vector<HostOp>& L = cherries.empty() ? hops : kept;
    const int nL = (int)L.size();
    // children from outside the list -- read at or before the first op that writes them, which may come later in the list
    // (such lists run in the caller's order): read as virtual cherries where the records can say so, i.e. when the list
    // never writes them, else as stored partials
    std::vector<int> vt1(readsVirtual ? in->nBuffers : 0, -1), vt2(readsVirtual ? in->nBuffers : 0, -1);
    for (const CherryRef& c : cherries) { vt1[c.buf] = c.tip1; vt2[c.buf] = c.tip2; }
    std::vector<CherryRef> external;
    {
        std::vector<char> seen(in->nBuffers, 0);
        for (int k = 0; k < n; ++k)
            for (int c : {hops[k].c1, hops[k].c2}) {
                if (firstWrite[c] < k || in->states32[c] != nullptr || seen[c]) continue;
                seen[c] = 1;
                const bool virt = readsVirtual && !written[c] && in->cherryTip1[c] >= 0;
                external.push_back(CherryRef{c, virt ? in->cherryTip1[c] : -1, virt ? in->cherryTip2[c] : -1});
                if (virt) { vt1[c] = in->cherryTip1[c]; vt2[c] = in->cherryTip2[c]; }
            }
    }
    CUDA_OK(storeExternal(in, external));
    {
        if (!byPartition) {
            if (preOrder) {
                if (in->prePhases) planPreorderPhases(hops, in->nBuffers, in->phaseT, wantSubsFor(in->Ppad), in->phaseTmin, in->phaseSmall, plan);
                else planLevels(hops, in->nBuffers, plan);
                for (Sub& sb : plan.subs) { sb.pBase = 0; sb.pLimit = in->Ppad; }
            }
        } else {
            // partitions are independent (disjoint pattern windows): plan each one on its own and merge the
            // plans phase by phase; every subtree carries its partition's pattern window
            std::vector<std::vector<int>> members(in->partitionCount);
            for (int k = 0; k < n; ++k) members[hops[k].part].push_back(k);
            std::vector<Plan> plans;
            std::vector<int> base;
            maxWindow = 1;
            for (int part = 0; part < in->partitionCount; ++part) {
                if (members[part].empty()) continue;
                std::vector<HostOp> sub(members[part].size());
                for (size_t q = 0; q < sub.size(); ++q) sub[q] = hops[members[part][q]];
                Plan pl;
                const int window = in->partEnd[part] - in->partBegin[part];
                if (sub[0].kind == 1 && in->prePhases) planPreorderPhases(sub, in->nBuffers, in->phaseT, wantSubsFor(std::max(1, window)), in->phaseTmin, in->phaseSmall, pl);
                else if (sub[0].kind == 1) planLevels(sub, in->nBuffers, pl);
                else planPhases(sub, in->nBuffers, in->reorder != 0, in->phaseT, wantSubsFor(std::max(1, window)), in->phaseTmin, in->phaseSmall, pl);
                base.push_back((int)plan.order.size());
                for (int idx : pl.order) plan.order.push_back(members[part][idx]);
                for (Sub& sb : pl.subs) {
                    sb.begin += base.back(); sb.end += base.back();
                    sb.pBase = in->partBegin[part]; sb.pLimit = in->partEnd[part];
                }
                maxWindow = std::max(maxWindow, window);
                plans.push_back(std::move(pl));
            }
            plan.phaseStart.assign(1, 0);
            for (size_t ph = 0;; ++ph) {
                bool any = false;
                for (const Plan& pl : plans) {
                    if (ph + 1 >= pl.phaseStart.size()) continue;
                    any = true;
                    for (int q = pl.phaseStart[ph]; q < pl.phaseStart[ph + 1]; ++q) plan.subs.push_back(pl.subs[q]);
                }
                if (!any) break;
                plan.phaseStart.push_back((int)plan.subs.size());
            }
        }
    }
    const std::vector<int>& order = plan.order;

    // ---- stack slots (4-state path only): one backward pass finds, for every produced value, the
    // position of its LAST reader inside this list (before the buffer is re-written); the forward
    // pass then parks results in slots and frees each slot at that last read.
    // The operand stack pays off where a phase is LATENCY-bound (few walks in flight: the tail of a full
    // evaluation, or the short dependent chain of an incremental update): it removes the store -> L2 -> load round
    // trip from every op of the chain.  Throughput-bound phases run without it (shared memory would cap occupancy).
    const bool stackEverywhere = fourState && in->walkVariant == 1 && !preOrder;
    const bool stackThin = fourState && in->walkVariant == 0 && in->stackTail && !preOrder;
    const int maxDepth = (stackEverywhere || stackThin) ? in->stackDepthMax : 0;
    const int nPhases = (int)plan.phaseStart.size() - 1;
    std::vector<char> subStack(plan.subs.size(), 0);
    std::vector<int> phaseDepth(std::max(nPhases, 1), 0), phaseOfSub(plan.subs.size(), 0);
    if (maxDepth > 0) {
        const int patsPerWarpS = (32 / in->matCP) * in->walkR;
        for (int ph = 0; ph < nPhases; ++ph) {
            long warps = 0;
            for (int q = plan.phaseStart[ph]; q < plan.phaseStart[ph + 1]; ++q) {
                warps += (plan.subs[q].pLimit - plan.subs[q].pBase + patsPerWarpS - 1) / patsPerWarpS;
                phaseOfSub[q] = ph;
            }
            const bool thin = warps < (long)in->smCount * 8;
            for (int q = plan.phaseStart[ph]; q < plan.phaseStart[ph + 1]; ++q) subStack[q] = stackEverywhere || thin;
        }
    }
    std::vector<int> lastReadOfProd(maxDepth > 0 ? nL : 0, -1);
    std::vector<int> subOfPos(nL, 0);
    for (int sIdx = 0; sIdx < (int)plan.subs.size(); ++sIdx)
        for (int q = plan.subs[sIdx].begin; q < plan.subs[sIdx].end; ++q) subOfPos[q] = sIdx;
    if (maxDepth > 0) {
        // per subtree: the stack is private to a (subtree, tile) walk
        std::vector<int> lastRead(in->nBuffers, -1);
        for (size_t sIdx = 0; sIdx < plan.subs.size(); ++sIdx) {
            if (!subStack[sIdx]) continue;
            const Sub& sb = plan.subs[sIdx];
            for (int pos = sb.end - 1; pos >= sb.begin; --pos) {
                const HostOp& o = L[order[pos]];
                lastReadOfProd[pos] = lastRead[o.dest];
                lastRead[o.dest] = -1;
                if (lastRead[o.c1] < 0) lastRead[o.c1] = pos;
                if (lastRead[o.c2] < 0) lastRead[o.c2] = pos;
            }
            for (int pos = sb.begin; pos < sb.end; ++pos) {      // leave no marks for the next subtree
                const HostOp& o = L[order[pos]];
                lastRead[o.dest] = lastRead[o.c1] = lastRead[o.c2] = -1;
            }
        }
    }
    std::vector<int> slotOf(maxDepth > 0 ? in->nBuffers : 0, -1), slotFreeAt(maxDepth > 0 ? in->nBuffers : 0, -1);
    std::vector<int> freeSlots;
    int depthUsed = 0, depthThisSub = 0, curSub = -1;

    const bool fourPath = in->matCP > 0;
    std::vector<CumGroup> cumGroups;
    std::vector<DevOp> dops(fourPath ? 0 : nL);
    std::vector<Op4> ops4(fourPath ? nL : 0);
    std::vector<int4> virtTips(readsVirtual ? nL : 0);     // k_walk4pv: the tips of each op's virtual children
    for (int pos = 0; pos < nL; ++pos) {
        const HostOp& o = L[order[pos]];
        const bool t1 = in->states32[o.c1] != nullptr;
        const bool t2 = in->states32[o.c2] != nullptr;
        int srcSlot1 = -1, srcSlot2 = -1, dstSlot = -1;
        if (maxDepth > 0 && subOfPos[pos] != curSub) {      // new subtree: fresh private stack
            curSub = subOfPos[pos];
            freeSlots.clear();
            depthThisSub = 0;
        }
        if (maxDepth > 0 && subStack[subOfPos[pos]]) {
            auto take = [&](int buf, bool isTip) -> int {
                if (isTip) return -1;
                const int slot = slotOf[buf];
                if (slot >= 0 && slotFreeAt[buf] == pos) { freeSlots.push_back(slot); slotOf[buf] = -1; }
                return slot;
            };
            srcSlot1 = take(o.c1, t1);
            srcSlot2 = (o.c2 == o.c1) ? srcSlot1 : take(o.c2, t2);
            if (slotOf[o.dest] >= 0) { freeSlots.push_back(slotOf[o.dest]); slotOf[o.dest] = -1; }   // stale value
            if (lastReadOfProd[pos] > pos) {         // a later op of this list reads the result
                int slot = -1;
                if (!freeSlots.empty()) { slot = freeSlots.back(); freeSlots.pop_back(); }
                else if (depthThisSub < maxDepth) {
                    slot = depthThisSub++;
                    depthUsed = std::max(depthUsed, depthThisSub);
                    phaseDepth[phaseOfSub[subOfPos[pos]]] = std::max(phaseDepth[phaseOfSub[subOfPos[pos]]], depthThisSub);
                }
                if (slot >= 0) { slotOf[o.dest] = slot; slotFreeAt[o.dest] = lastReadOfProd[pos]; dstSlot = slot; }
            }
        }
        const int pBegin = byPartition ? in->partBegin[o.part] : 0;
        const int pEnd = byPartition ? in->partEnd[o.part] : in->P;
        // In-list cumulative scaling (cumulativeScaleIndex != NONE) is NOT done inside the walk: independent subtrees of a
        // phase run concurrently over the same pattern columns, so a "cum[p] += log m" there would race.  The walk only
        // writes the per-node factors; one k_scale_accum launch per (cumulative buffer, pattern window) follows the phases.
        if (o.cum >= 0 && o.sw >= 0) {
            CumGroup* grp = nullptr;
            for (CumGroup& g : cumGroups) if (g.cum == o.cum && g.pBegin == pBegin && g.pEnd == pEnd) { grp = &g; break; }
            if (grp == nullptr) { cumGroups.push_back(CumGroup{o.cum, pBegin, pEnd, {}}); grp = &cumGroups.back(); }
            grp->indices.push_back(o.sw);
        }
        const int cum = -1;
        if (fourPath) {
            Op4& d = ops4[pos];
            // a virtual cherry child: its buffer index (recipe row) and its two tips
            const bool v1 = readsVirtual && !t1 && vt1[o.c1] >= 0, v2 = readsVirtual && !t2 && vt1[o.c2] >= 0;
            d.dest = in->slotOf[o.dest];
            d.c1 = t1 ? -(o.c1 + 1) : v1 ? o.c1 : in->slotOf[o.c1];
            d.c2 = t2 ? -(o.c2 + 1) : v2 ? o.c2 : in->slotOf[o.c2];
            d.m1 = o.m1; d.m2 = o.m2; d.sw = o.sw; d.sr = o.sr; d.cum = cum;
            d.pBegin = pBegin; d.pEnd = pEnd;
            d.slots = (unsigned)(srcSlot1 & 0xFF) | ((unsigned)(srcSlot2 & 0xFF) << 8) | ((unsigned)(dstSlot & 0xFF) << 16);
            d.pad_ = o.kind | (v1 ? 4 : 0) | (v2 ? 8 : 0);
            d.pfA = d.pfB = 0; d.pfM1 = d.pfM2 = -1;
            if (readsVirtual)
                virtTips[pos] = make_int4(v1 ? vt1[o.c1] : 0, v1 ? vt2[o.c1] : 0, v2 ? vt1[o.c2] : 0, v2 ? vt2[o.c2] : 0);
            if (in->forward && !(maxDepth > 0 && subStack[subOfPos[pos]]) && pos > plan.subs[subOfPos[pos]].begin)
                forwardFromPrevious(d, ops4[pos - 1], preOrder, readsVirtual ? &virtTips[pos] : nullptr);
        } else {
            DevOp& d = dops[pos];
            memset(&d, 0, sizeof d);
            d.dest = reinterpret_cast<double*>(in->partials[o.dest]);          // S > 4: always a double instance
            d.c1 = t1 ? nullptr : reinterpret_cast<const double*>(in->partials[o.c1]);
            d.c2 = t2 ? nullptr : reinterpret_cast<const double*>(in->partials[o.c2]);
            d.s1 = t1 ? (const void*)in->states32[o.c1] : nullptr;
            d.s2 = t2 ? (const void*)in->states32[o.c2] : nullptr;
            d.m1 = in->dMat + (size_t)o.m1 * in->matStride;
            d.m2 = in->dMat + (size_t)o.m2 * in->matStride;
            d.scaleWrite = o.sw >= 0 ? in->dScale + (size_t)o.sw * in->Ppad : nullptr;
            d.scaleRead = o.sr >= 0 ? in->dScale + (size_t)o.sr * in->Ppad : nullptr;
            d.cumScale = cum >= 0 ? in->dScale + (size_t)cum * in->Ppad : nullptr;
            d.pBegin = pBegin; d.pEnd = pEnd;
            d.srcSlot1 = d.srcSlot2 = d.dstSlot = -1;
            d.pad_ = o.kind;
            // register forwarding on the tensor-pipe walk (one category): the warp that wrote the previous op's 16-pattern
            // tile still holds it in its accumulators -- flag the child (moved to position 1; the product commutes exactly)
            if (in->forward && !preOrder && pos > plan.subs[subOfPos[pos]].begin) {
                const DevOp& pv = dops[pos - 1];
                if (pv.pBegin == d.pBegin && pv.pEnd == d.pEnd) {
                    if (d.c1 != nullptr && d.c1 == pv.dest) d.pad_ |= 2;
                    else if (d.c2 != nullptr && d.c2 == pv.dest) {
                        std::swap(d.c1, d.c2); std::swap(d.s1, d.s2); std::swap(d.m1, d.m2); d.pad_ |= 2;
                    }
                }
            }
        }
    }
    // sibling stack: lists whose phases the staged eigen walk may run (post-order, aligned, no matrix-form stack)
    std::vector<int> phaseSlots(std::max(nPhases, 1), 0);
    long fromStack = 0, fromMemory = 0;
    if (fourPath && eigenSlot >= 0 && !preOrder && !byPartition && maxDepth == 0 && in->stackSlots > 0 && walkStackBuilt(in)) {
        std::vector<int> subDepth;
        assignStackSlots(ops4, plan.subs, in->stackSlots, subDepth, fromStack, fromMemory);
        for (int ph = 0; ph < nPhases; ++ph)
            for (int q = plan.phaseStart[ph]; q < plan.phaseStart[ph + 1]; ++q) phaseSlots[ph] = std::max(phaseSlots[ph], subDepth[q]);
    }
    if (fourPath && in->lookahead && (!preOrder || in->lookaheadPre)) {
        // look-ahead fields: what op k+1 of the same walk will read from memory, except op k's own destination
        // only where the phase is throughput-bound; a thin phase is a pure latency chain and the extra instructions cost
        // more than the prefetch gives (measured on the 62-taxon benchmark2 alignment: +17 % with, in thin phases)
        std::vector<char> thick(plan.subs.size(), 0);
        const long perSub = (maxWindow + (32 / in->matCP) * in->walkR - 1) / ((32 / in->matCP) * in->walkR);
        for (int ph = 0; ph < nPhases; ++ph) {
            const bool t = (long)(plan.phaseStart[ph + 1] - plan.phaseStart[ph]) * perSub >= (long)in->smCount * 8;
            for (int q = plan.phaseStart[ph]; q < plan.phaseStart[ph + 1]; ++q) thick[q] = t;
        }
        for (size_t sIdx = 0; sIdx < plan.subs.size(); ++sIdx) {
            if ((maxDepth > 0 && subStack[sIdx]) || (!thick[sIdx] && in->lookahead < 2)) continue;
            for (int pos = plan.subs[sIdx].begin; pos + 1 < plan.subs[sIdx].end; ++pos) {
                Op4& d = ops4[pos];
                const Op4& nx = ops4[pos + 1];
                auto enc = [&](int child, bool fromRegisters, bool virt, bool fromStack) -> int {
                    if (fromRegisters || virt || fromStack) return 0;
                    if (child < 0) return ((-child - 1) << 1) | 1;
                    return child == d.dest ? 0 : ((child + 1) << 1);
                };
                d.pfA = enc(nx.c1, (nx.pad_ & 2) != 0, (nx.pad_ & 4) != 0, (nx.slots & 0xFF) != 0xFF);
                d.pfB = enc(nx.c2, false, (nx.pad_ & 8) != 0, ((nx.slots >> 8) & 0xFF) != 0xFF);
                if (d.pfA == 0) { d.pfA = d.pfB; d.pfB = 0; }
                d.pfM1 = nx.m1; d.pfM2 = nx.m2;
            }
        }
    }
    if (fourPath && getenv("B200_BEAGLE_DEBUG")) {
        int fwd = 0, internal = 0;
        for (const Op4& d : ops4) { fwd += (d.pad_ & 2) != 0; internal += (d.c1 >= 0) + (d.c2 >= 0); }
        fprintf(stderr, "[b200-beagle] plan: %d ops (%zu virtual cherries), %zu subtrees, %d phases, %d internal children, "
                "%d forwarded in registers, %ld read from the stack, %ld from memory\n", nL, cherries.size(), plan.subs.size(),
                nPhases, internal, fwd, fromStack, fromMemory);
    }
    // one block: [op records | subtree table | snapshot items], each part 256-byte aligned
    const size_t opBytes = (fourPath ? sizeof(Op4) : sizeof(DevOp)) * (size_t)nL;
    const size_t subBytes = sizeof(Sub) * plan.subs.size();
    const size_t snapBytes = sizeof(int4) * snap.size();
    const size_t subsOffset = (opBytes + 255) & ~size_t(255);
    const size_t snapOffset = subsOffset + ((subBytes + 255) & ~size_t(255));
    const size_t tipsBytes = sizeof(int4) * virtTips.size();
    const size_t tipsOffset = snapOffset + ((snapBytes + 255) & ~size_t(255));
    const size_t blockBytes = tipsOffset + tipsBytes;
    std::vector<char> hBlock(blockBytes, 0);
    memcpy(hBlock.data(), fourPath ? (const void*)ops4.data() : (const void*)dops.data(), opBytes);
    memcpy(hBlock.data() + subsOffset, plan.subs.data(), subBytes);
    if (snapBytes) memcpy(hBlock.data() + snapOffset, snap.data(), snapBytes);
    if (tipsBytes) memcpy(hBlock.data() + tipsOffset, virtTips.data(), tipsBytes);
    void* dOps = stage(in, hBlock.data(), blockBytes);
    void* tmp = nullptr;
    if (dOps == nullptr) {
        // list larger than the staging ring: one-off allocation
        CUDA_OK(cudaMalloc(&tmp, blockBytes));
        dOps = tmp;
        cudaError_t ce = cudaMemcpyAsync(dOps, hBlock.data(), blockBytes, cudaMemcpyHostToDevice, in->stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(in->stream);
        if (ce != cudaSuccess) { cudaFree(tmp); CUDA_OK(ce); }
    }
    void* dSubs = static_cast<char*>(dOps) + subsOffset;
    std::vector<int> depths(plan.phaseStart.size(), 0);
    for (size_t ph = 0; ph + 1 < plan.phaseStart.size(); ++ph) depths[ph] = (maxDepth > 0 && ph < phaseDepth.size()) ? phaseDepth[ph] : 0;
    cudaError_t e = launchPlan(in, dOps, dSubs, plan.phaseStart, depths, phaseSlots, fourPath, maxWindow, preOrder, eigenSlot, !byPartition,
                               static_cast<char*>(dOps) + snapOffset, (int)snap.size(),
                               readsVirtual ? static_cast<char*>(dOps) + tipsOffset : nullptr);
    if (e == cudaSuccess) e = accumulateInList(in, cumGroups);
    noteScaleWrites(in, hops);
    if (e == cudaSuccess) noteCherryWrites(in, hops, cherries);
    if (e == cudaSuccess && tmp == nullptr && in->planCacheSize > 0) {
        // remember the plan: device copy of the records (stream-ordered D2D out of the staging ring)
        if ((int)in->planCache.size() < in->planCacheSize) in->planCache.emplace_back();
        CachedPlan* slot = nullptr;            // first empty slot, else the least recently used entry
        for (CachedPlan& cp : in->planCache) {
            if (cp.dBlock == nullptr || cp.n < 0) { slot = &cp; break; }
            if (slot == nullptr || cp.lastUse < slot->lastUse) slot = &cp;
        }
        slot->dropGraph();
        slot->hits = 0;
        slot->graphFailed = false;
        slot->graphInvalidations = 0;
        if (slot->capacity < blockBytes) {
            if (slot->dBlock) cudaFree(slot->dBlock);
            slot->dBlock = nullptr; slot->capacity = 0;
            if (cudaMalloc(&slot->dBlock, blockBytes) == cudaSuccess) slot->capacity = blockBytes; else cudaGetLastError();
        }
        if (slot->dBlock != nullptr &&
            cudaMemcpyAsync(slot->dBlock, dOps, blockBytes, cudaMemcpyDeviceToDevice, in->stream) == cudaSuccess) {
            slot->key = hops; slot->n = n; slot->byPartition = byPartition; slot->epoch = in->bufferEpoch;
            slot->subsOffset = subsOffset; slot->snapOffset = snapOffset; slot->tipsOffset = tipsOffset;
            slot->cherries = cherries; slot->external = external; slot->readsVirtual = readsVirtual;
            slot->phaseStart = plan.phaseStart; slot->phaseDepth = depths;
            slot->phaseSlots = phaseSlots;
            slot->fourPath = fourPath; slot->maxWindow = maxWindow; slot->preOrder = preOrder;
            slot->lastUse = ++in->planClock;
            slot->cumGroups = cumGroups;
            slot->graphFailed = !cumGroups.empty();      // the accumulate launches stage fresh index arrays: never captured
        } else if (slot->dBlock != nullptr) {
            slot->n = -1;
        }
    }
    if (tmp != nullptr) { cudaStreamSynchronize(in->stream); cudaFree(tmp); }
    CUDA_OK(e);
    return BEAGLE_SUCCESS;
}

}  // namespace

namespace b200 {
Instance* instanceById(int id) { return getInstance(id); }
}

// ==============================================================================================
// exported C ABI
// ==============================================================================================
extern "C" {

#ifndef B200_SOURCE_HASH
#define B200_SOURCE_HASH "unhashed"
#endif
const char* beagleGetVersion(void) { return "4.0.1-b200+" B200_SOURCE_HASH; }
const char* b200GetSourceHash(void) { return B200_SOURCE_HASH; }

const char* beagleGetCitation(void) {
    return "H100-native tree-likelihood engine exposing the BEAGLE API.\n"
           "API after: Ayres et al. (2019) BEAGLE 3. Syst Biol 68:1052-1061.";
}

BeagleResourceList* beagleGetResourceList(void) {
    std::call_once(gResourceOnce, buildResources);
    return &gResourceList;
}

BeagleBenchmarkedResourceList* beagleGetBenchmarkedResourceList(
    int tipCount, int compactBufferCount, int stateCount, int patternCount, int categoryCount, int* resourceList,
    int resourceCount, long preferenceFlags, long requirementFlags, int eigenModelCount, int partitionCount,
    int calculateDerivatives, long benchmarkFlags);   // defined after the entry points it drives

int beagleCreateInstance(int tipCount, int partialsBufferCount, int compactBufferCount, int stateCount,
                         int patternCount, int eigenBufferCount, int matrixBufferCount, int categoryCount,
                         int scaleBufferCount, int* resourceList, int resourceCount, long preferenceFlags,
                         long requirementFlags, BeagleInstanceDetails* returnInfo) {
    if (tipCount < 0 || partialsBufferCount < 0 || compactBufferCount < 0 || stateCount < 2 ||
        patternCount < 1 || eigenBufferCount < 0 || matrixBufferCount < 0 || categoryCount < 1 ||
        scaleBufferCount < 0 || stateCount > 255)
        return BEAGLE_ERROR_OUT_OF_RANGE;
    if (requirementFlags & ~kSupportedFlags) return BEAGLE_ERROR_NO_RESOURCE;
    // storage precision: fp32 partials exist for the 4-state walk with C <= 8 (the range of the virtual cherries and the
    // fused incremental path); a single preference elsewhere is met with a double instance, a requirement is not met
    const bool singleFits = stateCount <= 4 && categoryCount <= 8;
    if (requirementFlags & BEAGLE_FLAG_PRECISION_SINGLE) {
        if (!singleFits || (requirementFlags & BEAGLE_FLAG_PRECISION_DOUBLE)) return BEAGLE_ERROR_NO_RESOURCE;
    }
    const bool single = singleFits && ((requirementFlags & BEAGLE_FLAG_PRECISION_SINGLE) ||
                                       ((preferenceFlags & BEAGLE_FLAG_PRECISION_SINGLE) &&
                                        !((preferenceFlags | requirementFlags) & BEAGLE_FLAG_PRECISION_DOUBLE)));
    BeagleResourceList* rl = beagleGetResourceList();
    int resource = -1;
    if (resourceList == nullptr || resourceCount <= 0) {
        if (rl->length > 1) resource = 1;
    } else {
        for (int k = 0; k < resourceCount; ++k)
            if (resourceList[k] >= 1 && resourceList[k] < rl->length) { resource = resourceList[k]; break; }
    }
    if (resource < 1) return BEAGLE_ERROR_NO_RESOURCE;   // no CUDA device, or only resource 0 requested

    if (resource == gShardResource) {
        // one instance over several GPUs: the shards are ordinary instances, this id only forwards (multi.cu)
        Instance* parent = new Instance();
        parent->resource = resource;
        parent->device = gShardDevices[0];
        parent->P = patternCount; parent->S = stateCount; parent->C = categoryCount; parent->tipCount = tipCount;
        const int g = (int)gShardDevices.size();
        const int rc = shardedCreate(parent, g, gShardDevices.data(), tipCount, partialsBufferCount, compactBufferCount,
                                     stateCount, patternCount, eigenBufferCount, matrixBufferCount, categoryCount,
                                     scaleBufferCount, preferenceFlags, requirementFlags, returnInfo);
        if (rc != BEAGLE_SUCCESS) { delete parent; return rc; }
        if (returnInfo != nullptr) {
            returnInfo->resourceNumber = resource;
            returnInfo->resourceName = rl->list[resource].name;
            parent->flags = returnInfo->flags;
        }
        std::lock_guard<std::mutex> lock(gMutex);
        int id = -1;
        for (size_t k = 0; k < gInstances.size(); ++k) if (gInstances[k] == nullptr) { id = (int)k; break; }
        if (id < 0) { gInstances.push_back(nullptr); id = (int)gInstances.size() - 1; }
        gInstances[id] = parent;
        parent->id = id;
        return id;
    }

    Instance* in = new Instance();
    in->device = resource - 1;
    in->resource = resource;
    if (cudaSetDevice(in->device) != cudaSuccess) { delete in; return BEAGLE_ERROR_NO_RESOURCE; }
    in->tipCount = tipCount; in->nPartials = partialsBufferCount; in->nCompact = compactBufferCount;
    in->S = stateCount; in->P = patternCount; in->nEigen = eigenBufferCount; in->nMatrices = matrixBufferCount;
    in->C = categoryCount; in->nScale = scaleBufferCount;
    in->Sp = stateCount <= 4 ? 4 : ((stateCount + 7) / 8) * 8;      // multiples of the 8x8x4 DMMA tile
    in->Ppad = ((patternCount + 31) / 32) * 32;
    in->nBuffers = partialsBufferCount + compactBufferCount;
    in->nSets = std::max(1, eigenBufferCount);
    in->single = single;
    in->complexEigen = (requirementFlags | preferenceFlags) & BEAGLE_FLAG_EIGEN_COMPLEX;
    in->logScalers = (requirementFlags | preferenceFlags) & BEAGLE_FLAG_SCALERS_LOG;
    in->flags = (single ? BEAGLE_FLAG_PRECISION_SINGLE : BEAGLE_FLAG_PRECISION_DOUBLE) | BEAGLE_FLAG_COMPUTATION_SYNCH |
                BEAGLE_FLAG_SCALING_MANUAL |
                BEAGLE_FLAG_VECTOR_NONE | BEAGLE_FLAG_THREADING_NONE | BEAGLE_FLAG_PROCESSOR_GPU |
                BEAGLE_FLAG_FRAMEWORK_CUDA | BEAGLE_FLAG_PARALLELOPS_GRID |
                (in->complexEigen ? BEAGLE_FLAG_EIGEN_COMPLEX : BEAGLE_FLAG_EIGEN_REAL) |
                (in->logScalers ? BEAGLE_FLAG_SCALERS_LOG : BEAGLE_FLAG_SCALERS_RAW);
    if ((requirementFlags | preferenceFlags) & BEAGLE_FLAG_PREORDER_TRANSPOSE_AUTO) in->flags |= BEAGLE_FLAG_PREORDER_TRANSPOSE_AUTO;
    if ((requirementFlags | preferenceFlags) & BEAGLE_FLAG_SCALING_DYNAMIC) {
        in->flags &= ~BEAGLE_FLAG_SCALING_MANUAL;
        in->flags |= BEAGLE_FLAG_SCALING_DYNAMIC;
    }
    in->partialsElems = (size_t)in->C * in->Ppad * in->Sp;
    if (in->Sp == 4 && in->C <= 32) {
        int cp = 1;
        while (cp < in->C) cp <<= 1;
        in->matCP = cp;
        in->matStride = (size_t)16 * cp + 52 * (size_t)in->C;     // [j][CP][i] + Mpad[c][8][4] + MTg[c][5][4]
        in->matStride = (in->matStride + 3) & ~size_t(3);        // keep every buffer 32-byte aligned
    } else {
        in->matCP = 0;
        // MT[c][j][i] (FMA walk, tip gathers), then the tensor-path operands with an (Sp+4)-double row stride so that ONE
        // contiguous bulk copy lands them in shared memory bank-conflict free: M[c][i][.] and MT[c][j][.]
        in->matStride = (size_t)in->C * in->Sp * (in->Sp + 2 * (size_t)(in->Sp + 4));
    }
    in->slotOf.assign(in->nBuffers, -1);
    in->partials.assign(in->nBuffers, nullptr);
    in->states8.assign(in->nBuffers, nullptr);
    in->states32.assign(in->nBuffers, nullptr);
    in->scaleIsLog.assign(std::max(1, in->nScale), in->logScalers ? 1 : 0);
    in->matEigen.assign(std::max(1, in->nMatrices), -1);
    in->matEigenGen.assign(std::max(1, in->nMatrices), 0u);
    in->eigenGen.assign(std::max(1, in->nEigen), 0u);
    in->eigenReal.assign(std::max(1, in->nEigen), 0);
    in->eigenKind.assign(std::max(1, in->nEigen), 0);
    in->hEigen.assign((size_t)std::max(1, in->nEigen) * 36, 0.0);
    in->eigenWalk = envInt("B200_EIGEN_WALK", 1);
    in->tipMode = envInt("B200_TIP_MODE", 3);
    in->thinTipMode = envInt("B200_THIN_TIP_MODE", in->tipMode);
    in->virtualCherries = envInt("B200_VIRTUAL_CHERRIES", 1);
    in->walkBlock = 128;
    in->walkVariant = envInt("B200_WALK_VARIANT", 0);
    in->reorder = envInt("B200_REORDER", 1);
    in->forward = envInt("B200_FORWARD", 1);
    in->stackSlots = envInt("B200_WALK_STACK_SLOTS", 1) != 0 ? kStackSlots : 0;
    in->debugLog = getenv("B200_BEAGLE_DEBUG") != nullptr;
    in->lookahead = envInt("B200_LOOKAHEAD", 1);
    in->useGraphs = envInt("B200_GRAPHS", 1);
    in->prePhases = envInt("B200_PRE_PHASES", 1);
    in->lookaheadPre = envInt("B200_LOOKAHEAD_PRE", 1);
    in->planCacheSize = std::max(0, std::min(16, envInt("B200_PLAN_CACHE", 4)));
    in->planCache.reserve(16);
    in->thinR1 = envInt("B200_THIN_R1", 1);
    in->stackTail = envInt("B200_STACK_TAIL", 0);     // measured slower (0.458 vs 0.436 ms): off by default
    in->phaseT = envInt("B200_PHASE_T", 0);
    in->phaseTmin = std::max(1, envInt("B200_PHASE_TMIN", 4));
    in->phaseSmall = envInt("B200_PHASE_SMALL", 24);
    in->phaseOversub = std::max(0, envInt("B200_PHASE_OVERSUB", 0));      // 0 = by subtree width (see wantSubsFor)
    in->walkMinBlocks = envInt("B200_WALK_MINB", 4);
    in->walkMinBlocksSet = getenv("B200_WALK_MINB") != nullptr;
    in->tensorR = envInt("B200_TENSOR_R", 2) >= 4 ? 4 : 2;
    in->genericMma = envInt("B200_GENERIC_MMA", 1);
    in->mmaWarps = envInt("B200_MMA_WARPS", 4) == 8 ? 8 : 4;     // 8 = 256-thread blocks with cp.async double buffering
    // the SM count sizes the walk below: query the device first
    cudaDeviceProp prop;
    bool ok = cudaGetDeviceProperties(&prop, in->device) == cudaSuccess;
    if (ok) { in->smCount = prop.multiProcessorCount; in->maxSmemOptin = prop.sharedMemPerBlockOptin; }
    in->walkR = envInt("B200_WALK_R", 4);
    if (in->walkR != 1 && in->walkR != 2 && in->walkR != 4 && in->walkR != 8) in->walkR = 4;
    if (getenv("B200_WALK_R") == nullptr && in->matCP > 0) {
        // patterns per thread: as many as still leave >= 1 warp per SM inside ONE subtree walk (the phases supply the rest of
        // the parallelism: measured on the 6000-pattern Makona-like set, 25 subtrees per launch: R = 4 0.273 ms, R = 2 0.340 ms)
        const int G = 32 / in->matCP;
        while (in->walkR > 1 && (in->Ppad + G * in->walkR - 1) / (G * in->walkR) < in->smCount) in->walkR >>= 1;
    }
    in->stackDepthMax = std::min(64, std::max(0, envInt("B200_STACK_DEPTH", 12)));
    if (single) { in->walkVariant = 0; in->stackTail = 0; }     // the experimental walk variants are built for fp64 only

    ok = ok && cudaStreamCreateWithFlags(&in->stream, cudaStreamNonBlocking) == cudaSuccess;
    const size_t eigenStride = 2 * (size_t)in->S * in->S + 2 * in->S;
    const size_t matElems = (size_t)in->nMatrices * in->matStride;
    const int rootBlocks = (in->Ppad + 255) / 256;
    in->stageSize = size_t(8) << 20;
    auto alloc = [&](auto** p, size_t elems) {
        if (!ok) return;
        using T = std::remove_pointer_t<std::remove_pointer_t<decltype(p)>>;
        size_t bytes = std::max<size_t>(elems, 1) * sizeof(T);
        ok = cudaMalloc(reinterpret_cast<void**>(p), bytes) == cudaSuccess &&
             cudaMemsetAsync(*p, 0, bytes, in->stream) == cudaSuccess;
    };
    alloc(&in->dEigen, std::max(1, in->nEigen) * eigenStride);
    alloc(&in->dMat, matElems);
    if (in->matCP > 0) alloc(&in->dEvec, (size_t)in->nMatrices * in->matCP * 4);
    if (in->matCP > 0 && in->matCP <= 8 && in->virtualCherries) {
        alloc(&in->dRecipe, (size_t)in->nBuffers * 32 * in->matCP);
        in->cherryTip1.assign(in->nBuffers, -1);
        in->cherryTip2.assign(in->nBuffers, -1);
        in->cherryStored.assign(in->nBuffers, 0);
    }
    if (in->matCP > 0 && in->matCP <= 8) {
        alloc(&in->dIncSums, (size_t)in->Ppad / 4 + 8);
        alloc(&in->dIncCounter, 4);
        in->fuseSmall = envInt("B200_FUSE", 1);
        if (ok && in->fuseSmall) {
            // the fused evaluation lands its result here; without mapped memory the fusion is simply off
            if (cudaHostAlloc(reinterpret_cast<void**>(&in->hMapped), 64, cudaHostAllocMapped) == cudaSuccess &&
                cudaHostGetDevicePointer(reinterpret_cast<void**>(&in->dMapped), in->hMapped, 0) == cudaSuccess) {
                memset(in->hMapped, 0, 64);
            } else {
                cudaGetLastError();
                if (in->hMapped) cudaFreeHost(in->hMapped);
                in->hMapped = nullptr;
            }
        }
    }
    alloc(&in->dRates, (size_t)in->nSets * in->C);
    alloc(&in->dWeights, (size_t)in->nSets * in->C);
    alloc(&in->dFreqs, (size_t)in->nSets * in->Sp);
    alloc(&in->dScale, (size_t)in->nScale * in->Ppad);
    alloc(&in->dPatternWeights, in->Ppad);
    alloc(&in->dPatternPartitions, in->Ppad);
    alloc(&in->dSite, in->Ppad);
    alloc(&in->dBlockSums, rootBlocks);
    alloc(&in->dOut, 1024);
    alloc(&in->dCounter, 4);
    alloc(&in->dStage, in->stageSize);
    alloc(&in->states8Base, (size_t)std::max(1, in->tipCount) * in->Ppad);
    alloc(&in->states32Base, (size_t)std::max(1, in->tipCount) * in->Ppad);
    if (ok) {
        // every partials buffer the caller may address, else (memory-tight) all but the compact tips
        int want[2] = {in->nPartials, std::max(1, in->nPartials - std::min(in->nCompact, in->tipCount))};
        for (int attempt = 0; attempt < 2 && in->partialsBase == nullptr; ++attempt) {
            size_t bytes = (size_t)want[attempt] * in->partialsElems * in->elemBytes();
            if (cudaMalloc(reinterpret_cast<void**>(&in->partialsBase), bytes) == cudaSuccess) in->nSlots = want[attempt];
            else { cudaGetLastError(); in->partialsBase = nullptr; }
        }
        if (in->partialsBase == nullptr) { destroyInstance(in); return BEAGLE_ERROR_OUT_OF_MEMORY; }
    }
    ok = ok && cudaMallocHost(reinterpret_cast<void**>(&in->hStage), in->stageSize) == cudaSuccess;
    ok = ok && cudaHostGetDevicePointer(reinterpret_cast<void**>(&in->hStageDev), in->hStage, 0) == cudaSuccess;
    ok = ok && cudaMallocHost(reinterpret_cast<void**>(&in->hOut), 1024 * sizeof(double)) == cudaSuccess;
    if (ok) {
        // default: one rate category set of all ones, unit pattern weights (upstream defaults)
        in->hRates.assign((size_t)in->nSets * in->C, 1.0);
        in->hWeights.assign((size_t)in->nSets * in->C, 0.0);
        in->hFreqs.assign((size_t)in->nSets * 4, 0.0);
        std::vector<double> ones((size_t)std::max(in->nSets * in->C, in->Ppad), 1.0);
        ok = cudaMemcpyAsync(in->dRates, ones.data(), sizeof(double) * in->nSets * in->C, cudaMemcpyHostToDevice,
                             in->stream) == cudaSuccess;
        std::vector<double> w(in->Ppad, 0.0);
        std::fill(w.begin(), w.begin() + in->P, 1.0);
        ok = ok && cudaMemcpyAsync(in->dPatternWeights, w.data(), sizeof(double) * in->Ppad, cudaMemcpyHostToDevice,
                                   in->stream) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(in->stream) == cudaSuccess;
    }
    if (!ok) {
        cudaError_t e = cudaGetLastError();
        destroyInstance(in);
        return e == cudaErrorMemoryAllocation ? BEAGLE_ERROR_OUT_OF_MEMORY : BEAGLE_ERROR_GENERAL;
    }
    in->partitionCount = 1;
    in->partBegin.assign(1, 0);
    in->partEnd.assign(1, in->P);
    {
        std::lock_guard<std::mutex> lock(gMutex);
        int id = -1;
        for (size_t k = 0; k < gInstances.size(); ++k) if (gInstances[k] == nullptr) { id = (int)k; break; }
        if (id < 0) { gInstances.push_back(nullptr); id = (int)gInstances.size() - 1; }
        gInstances[id] = in;
        in->id = id;
    }
    if (returnInfo != nullptr) {
        returnInfo->resourceNumber = resource;
        returnInfo->resourceName = rl->list[resource].name;
        returnInfo->implName = single ? gImplNameSingle : gImplName;
        returnInfo->implDescription = gImplDesc;
        returnInfo->flags = in->flags;
    }
    return in->id;
}

int beagleFinalizeInstance(int instance) {
    Instance* in = nullptr;
    {
        std::lock_guard<std::mutex> lock(gMutex);
        if (instance < 0 || instance >= (int)gInstances.size() || gInstances[instance] == nullptr)
            return BEAGLE_ERROR_UNINITIALIZED_INSTANCE;
        in = gInstances[instance];
        gInstances[instance] = nullptr;
    }
    destroyInstance(in);
    return BEAGLE_SUCCESS;
}

int beagleFinalize(void) {
    std::vector<Instance*> all;
    {
        std::lock_guard<std::mutex> lock(gMutex);
        all.swap(gInstances);
    }
    for (Instance* in : all) if (in) destroyInstance(in);
    return BEAGLE_SUCCESS;
}

int beagleSetCPUThreadCount(int instance, int) {
    SH(instance, BEAGLE_SUCCESS);
    GET_INSTANCE(in, instance);
    (void)in;
    return BEAGLE_SUCCESS;
}

// ---- data upload ------------------------------------------------------------------------------
int beagleSetTipStates(int instance, int tipIndex, const int* inStates) {
    SH(instance, shSetTipStates(sh, tipIndex, inStates));
    GET_INSTANCE(in, instance);
    if (!validRange(tipIndex, in->nBuffers) || inStates == nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<int> s32(in->Ppad, in->S);
    std::vector<uint8_t> s8(in->Ppad, (uint8_t)in->S);
    for (int p = 0; p < in->P; ++p) {
        int s = inStates[p];
        if (s < 0 || s >= in->S) s = in->S;
        s32[p] = s;
        s8[p] = (uint8_t)s;
    }
    if (tipIndex >= in->tipCount) return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(settleCherriesOf(in, tipIndex));      // cherries computed from the old states keep their values
    in->states32[tipIndex] = in->states32Base + (size_t)tipIndex * in->Ppad;
    in->states8[tipIndex] = in->states8Base + (size_t)tipIndex * in->Ppad;
    CUDA_OK(cudaMemcpyAsync(in->states32[tipIndex], s32.data(), sizeof(int) * in->Ppad, cudaMemcpyHostToDevice, in->stream));
    CUDA_OK(cudaMemcpyAsync(in->states8[tipIndex], s8.data(), in->Ppad, cudaMemcpyHostToDevice, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    // the buffer is a compact tip from now on (states32[idx] != nullptr marks it; a previously assigned
    // partials slot stays reserved)
    in->bufferEpoch++;
    return BEAGLE_SUCCESS;
}

int beagleGetTipStates(int instance, int tipIndex, int* outStates) {
    SH(instance, shGetTipStates(sh, tipIndex, outStates));
    GET_INSTANCE(in, instance);
    if (!validRange(tipIndex, in->nBuffers) || in->states32[tipIndex] == nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(cudaMemcpyAsync(outStates, in->states32[tipIndex], sizeof(int) * in->P, cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    return BEAGLE_SUCCESS;
}

static int setPartialsImpl(Instance* in, int bufferIndex, const double* inPartials, bool perCategory) {
    if (!validRange(bufferIndex, in->nBuffers) || inPartials == nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
    char* dst = ensurePartials(in, bufferIndex);
    if (dst == nullptr) return BEAGLE_ERROR_OUT_OF_MEMORY;
    CUDA_OK(settleCherriesOf(in, bufferIndex));
    if (!in->cherryTip1.empty()) in->cherryTip1[bufferIndex] = -1;
    std::vector<double> tmp(in->partialsElems, 0.0);
    for (int c = 0; c < in->C; ++c)
        for (int p = 0; p < in->Ppad; ++p) {
            double* row = tmp.data() + ((size_t)c * in->Ppad + p) * in->Sp;
            if (p < in->P) {
                const double* src = inPartials + ((size_t)(perCategory ? c : 0) * in->P + p) * in->S;
                for (int i = 0; i < in->S; ++i) row[i] = src[i];
            } else {
                for (int i = 0; i < in->S; ++i) row[i] = 1.0;     // padded patterns: harmless, finite
            }
        }
    if (in->single) {
        // fp32 storage: the rounding of the walk kernels (walk4.cuh roundCell), a subnormal result becomes a signed zero
        std::vector<float> narrow(in->partialsElems);
        for (size_t q = 0; q < narrow.size(); ++q) {
            const float f = (float)tmp[q];
            narrow[q] = std::fpclassify(f) == FP_SUBNORMAL ? std::copysign(0.0f, f) : f;
        }
        CUDA_OK(cudaMemcpyAsync(dst, narrow.data(), sizeof(float) * narrow.size(), cudaMemcpyHostToDevice, in->stream));
        CUDA_OK(cudaStreamSynchronize(in->stream));
    } else {
        CUDA_OK(cudaMemcpyAsync(dst, tmp.data(), sizeof(double) * in->partialsElems, cudaMemcpyHostToDevice, in->stream));
        CUDA_OK(cudaStreamSynchronize(in->stream));
    }
    if (in->states32[bufferIndex] != nullptr) in->bufferEpoch++;      // tip -> partials: cached plans are stale
    in->states32[bufferIndex] = nullptr;
    in->states8[bufferIndex] = nullptr;
    return BEAGLE_SUCCESS;
}

int beagleSetTipPartials(int instance, int tipIndex, const double* inPartials) {
    SH(instance, shSetPartials(sh, tipIndex, inPartials, false));
    GET_INSTANCE(in, instance);
    return setPartialsImpl(in, tipIndex, inPartials, false);
}

int beagleSetPartials(int instance, int bufferIndex, const double* inPartials) {
    SH(instance, shSetPartials(sh, bufferIndex, inPartials, true));
    GET_INSTANCE(in, instance);
    return setPartialsImpl(in, bufferIndex, inPartials, true);
}

int beagleGetPartials(int instance, int bufferIndex, int scaleIndex, double* outPartials) {
    SH(instance, shGetPartials(sh, bufferIndex, scaleIndex, outPartials));
    GET_INSTANCE(in, instance);
    if (!validRange(bufferIndex, in->nBuffers) || in->partials[bufferIndex] == nullptr || outPartials == nullptr)
        return BEAGLE_ERROR_OUT_OF_RANGE;
    if (scaleIndex != BEAGLE_OP_NONE && !validRange(scaleIndex, in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(storeCherries(in, &bufferIndex, 1));
    std::vector<double> tmp(in->partialsElems);
    const double* src = reinterpret_cast<const double*>(in->partials[bufferIndex]);
    double* dTmp = nullptr;
    if (in->single) {
        // fp32 storage: widen here; with a scale index the fp64 unscaling below then runs on the widened copy
        std::vector<float> narrow(in->partialsElems);
        CUDA_OK(cudaMemcpyAsync(narrow.data(), in->partials[bufferIndex], sizeof(float) * narrow.size(),
                                cudaMemcpyDeviceToHost, in->stream));
        CUDA_OK(cudaStreamSynchronize(in->stream));
        for (size_t q = 0; q < narrow.size(); ++q) tmp[q] = narrow[q];
    }
    if (scaleIndex != BEAGLE_OP_NONE) {
        CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&dTmp), sizeof(double) * in->partialsElems));
        if (in->single) {
            const cudaError_t eUp = cudaMemcpyAsync(dTmp, tmp.data(), sizeof(double) * in->partialsElems,
                                                    cudaMemcpyHostToDevice, in->stream);
            if (eUp != cudaSuccess) { cudaFree(dTmp); CUDA_OK(eUp); }
        } else {
            CUDA_OK(cudaMemcpyAsync(dTmp, src, sizeof(double) * in->partialsElems, cudaMemcpyDeviceToDevice, in->stream));
        }
        CUDA_OK(launchRescalePartialsForGet(in, dTmp, in->dScale + (size_t)scaleIndex * in->Ppad));
        src = dTmp;
    }
    cudaError_t e = cudaSuccess;
    if (!in->single || dTmp != nullptr) {          // a single instance without a scale index has tmp already
        e = cudaMemcpyAsync(tmp.data(), src, sizeof(double) * in->partialsElems, cudaMemcpyDeviceToHost, in->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(in->stream);
    }
    if (dTmp) cudaFree(dTmp);
    CUDA_OK(e);
    for (int c = 0; c < in->C; ++c)
        for (int p = 0; p < in->P; ++p)
            memcpy(outPartials + ((size_t)c * in->P + p) * in->S, tmp.data() + ((size_t)c * in->Ppad + p) * in->Sp,
                   sizeof(double) * in->S);
    return BEAGLE_SUCCESS;
}

int beagleSetEigenDecomposition(int instance, int eigenIndex, const double* inEigenVectors,
                                const double* inInverseEigenVectors, const double* inEigenValues) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleSetEigenDecomposition(c, eigenIndex, inEigenVectors, inInverseEigenVectors, inEigenValues); }));
    GET_INSTANCE(in, instance);
    if (!validRange(eigenIndex, in->nEigen)) return BEAGLE_ERROR_OUT_OF_RANGE;
    const size_t S = in->S, stride = 2 * S * S + 2 * S;
    std::vector<double> pack(stride, 0.0);
    memcpy(pack.data(), inEigenVectors, sizeof(double) * S * S);
    memcpy(pack.data() + S * S, inInverseEigenVectors, sizeof(double) * S * S);
    memcpy(pack.data() + 2 * S * S, inEigenValues, sizeof(double) * (in->complexEigen ? 2 * S : S));
    bool realSystem = true;
    if (in->complexEigen) for (size_t k = 0; k < S; ++k) realSystem = realSystem && inEigenValues[S + k] == 0.0;
    in->eigenKind[eigenIndex] = realSystem ? 1 : 2;
    if (in->matCP > 0) {
        // host copy for the eigen-form walk (V, V^-1 travel by value in its launch); the generation only moves when the
        // content does, so that re-uploading an unchanged system keeps captured graphs valid
        double h[36] = {0.0};                 // V | V^-1 | eigenvalues (compared, not passed on)
        for (size_t k = 0; k < S; ++k) h[32 + k] = inEigenValues[k];
        for (size_t i = 0; i < S; ++i)
            for (size_t k = 0; k < S; ++k) { h[4 * i + k] = inEigenVectors[i * S + k]; h[16 + 4 * i + k] = inInverseEigenVectors[i * S + k]; }
        bool real = true;
        if (in->complexEigen) for (size_t k = 0; k < S; ++k) real = real && inEigenValues[S + k] == 0.0;
        double* dst = in->hEigen.data() + (size_t)eigenIndex * 36;
        if (memcmp(dst, h, sizeof h) != 0 || in->eigenGen[eigenIndex] == 0 || (bool)in->eigenReal[eigenIndex] != real) {
            memcpy(dst, h, sizeof h);
            in->eigenGen[eigenIndex]++;
        }
        in->eigenReal[eigenIndex] = real ? 1 : 0;
    }
    return uploadSmall(in, in->dEigen + (size_t)eigenIndex * stride, pack.data(), sizeof(double) * stride);
}

int beagleSetStateFrequencies(int instance, int stateFrequenciesIndex, const double* inStateFrequencies) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleSetStateFrequencies(c, stateFrequenciesIndex, inStateFrequencies); }));
    GET_INSTANCE(in, instance);
    if (!validRange(stateFrequenciesIndex, in->nSets)) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<double> f(in->Sp, 0.0);
    memcpy(f.data(), inStateFrequencies, sizeof(double) * in->S);
    if (in->hFreqs.size() == (size_t)in->nSets * 4 && in->S <= 4)          // host mirror: travels by value in the fused launch
        for (int i = 0; i < 4; ++i) in->hFreqs[(size_t)stateFrequenciesIndex * 4 + i] = i < in->S ? inStateFrequencies[i] : 0.0;
    return uploadSmall(in, in->dFreqs + (size_t)stateFrequenciesIndex * in->Sp, f.data(), sizeof(double) * in->Sp);
}

int beagleSetCategoryWeights(int instance, int categoryWeightsIndex, const double* inCategoryWeights) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleSetCategoryWeights(c, categoryWeightsIndex, inCategoryWeights); }));
    GET_INSTANCE(in, instance);
    if (!validRange(categoryWeightsIndex, in->nSets)) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::copy(inCategoryWeights, inCategoryWeights + in->C, in->hWeights.begin() + (size_t)categoryWeightsIndex * in->C);
    return uploadSmall(in, in->dWeights + (size_t)categoryWeightsIndex * in->C, inCategoryWeights, sizeof(double) * in->C);
}

int beagleSetCategoryRatesWithIndex(int instance, int categoryRatesIndex, const double* inCategoryRates) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleSetCategoryRatesWithIndex(c, categoryRatesIndex, inCategoryRates); }));
    GET_INSTANCE(in, instance);
    if (!validRange(categoryRatesIndex, in->nSets)) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::copy(inCategoryRates, inCategoryRates + in->C, in->hRates.begin() + (size_t)categoryRatesIndex * in->C);
    return uploadSmall(in, in->dRates + (size_t)categoryRatesIndex * in->C, inCategoryRates, sizeof(double) * in->C);
}

int beagleSetCategoryRates(int instance, const double* inCategoryRates) {
    return beagleSetCategoryRatesWithIndex(instance, 0, inCategoryRates);
}

int beagleSetPatternWeights(int instance, const double* inPatternWeights) {
    SH(instance, shSetPatternWeights(sh, inPatternWeights));
    GET_INSTANCE(in, instance);
    std::vector<double> w(in->Ppad, 0.0);
    memcpy(w.data(), inPatternWeights, sizeof(double) * in->P);
    CUDA_OK(cudaMemcpyAsync(in->dPatternWeights, w.data(), sizeof(double) * in->Ppad, cudaMemcpyHostToDevice, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    return BEAGLE_SUCCESS;
}

int beagleSetPatternPartitions(int instance, int partitionCount, const int* inPatternPartitions) {
    SH(instance, BEAGLE_ERROR_NO_IMPLEMENTATION);
    GET_INSTANCE(in, instance);
    if (partitionCount < 1 || partitionCount > 1000) return BEAGLE_ERROR_OUT_OF_RANGE;
    // contiguous, non-decreasing maps only -- what MPDLD:520-533 builds
    std::vector<int> begin(partitionCount, 0), end(partitionCount, 0);
    int prev = -1;
    for (int p = 0; p < in->P; ++p) {
        int k = inPatternPartitions[p];
        if (k < 0 || k >= partitionCount) return BEAGLE_ERROR_OUT_OF_RANGE;
        if (k < prev) return BEAGLE_ERROR_NO_IMPLEMENTATION;
        if (k != prev) { for (int q = prev + 1; q <= k; ++q) begin[q] = end[q] = p; prev = k; }
        end[k] = p + 1;
    }
    for (int q = prev + 1; q < partitionCount; ++q) begin[q] = end[q] = in->P;
    in->bufferEpoch++;
    in->partitionCount = partitionCount;
    in->partBegin = begin;
    in->partEnd = end;
    in->hostPartitions.assign(inPatternPartitions, inPatternPartitions + in->P);
    return BEAGLE_SUCCESS;
}

// ---- transition matrices ----------------------------------------------------------------------
static int updateMatricesImpl(Instance* in, const int* eigenIndices, int eigenIndexScalar, const int* rateSets,
                              const int* probabilityIndices, const double* edgeLengths, int count) {
    if (count <= 0) return BEAGLE_SUCCESS;
    // one staged block = one H2D copy: [edge lengths (count doubles)][matrix, eigen, rate-set indices (3 count ints)]
    std::vector<double> block((size_t)count + (3 * (size_t)count + 1) / 2);
    int* pack = reinterpret_cast<int*>(block.data() + count);
    for (int k = 0; k < count; ++k) {
        int e = eigenIndices ? eigenIndices[k] : eigenIndexScalar;
        int r = rateSets ? rateSets[k] : 0;
        if (!validRange(probabilityIndices[k], in->nMatrices) || !validRange(e, in->nEigen) ||
            !validRange(r, in->nSets))
            return BEAGLE_ERROR_OUT_OF_RANGE;
        pack[k] = probabilityIndices[k];
        pack[count + k] = e;
        pack[2 * (size_t)count + k] = r;
    }
    if (in->matCP > 0)
        for (int k = 0; k < count; ++k) {
            const int e = eigenIndices ? eigenIndices[k] : eigenIndexScalar;
            in->matEigen[probabilityIndices[k]] = e;
            in->matEigenGen[probabilityIndices[k]] = in->eigenGen[e];
        }
    memcpy(block.data(), edgeLengths, sizeof(double) * count);
    // 4-state: k_transition4 reads the block in place over PCIe, so no copy, and no wait for one, precedes the kernel
    // (measured on cfg 2: the copy took 3.4 us and the kernel started 2-8 us after it)
    const size_t blockBytes = sizeof(double) * block.size();
    const double* dLen = static_cast<const double*>(in->matCP > 0 ? stageMapped(in, block.data(), blockBytes)
                                                                   : stage(in, block.data(), blockBytes));
    if (dLen == nullptr) return BEAGLE_ERROR_OUT_OF_MEMORY;
    const int* dIdx = reinterpret_cast<const int*>(dLen + count);
    TimedScope ts(in, T_MATRICES);
    CUDA_OK(launchTransitionMatrices(in, dIdx, dIdx + count, dIdx + 2 * (size_t)count, dLen, count));
    return BEAGLE_SUCCESS;
}

// ---- deferred small evaluations (incr.cu) --------------------------------------------------------------------------
}  // extern "C"
namespace {
int flushPendingImpl(Instance* in) {
    int rc = BEAGLE_SUCCESS;
    if (!in->pendingMats.empty()) {
        const int n = (int)in->pendingMats.size();
        std::vector<int> eig(n), rate(n), prob(n);
        std::vector<double> len(n);
        for (int k = 0; k < n; ++k) {
            eig[k] = in->pendingMats[k].eigen; rate[k] = in->pendingMats[k].rateSet;
            prob[k] = in->pendingMats[k].prob; len[k] = in->pendingMats[k].len;
        }
        in->pendingMats.clear();
        rc = updateMatricesImpl(in, eig.data(), 0, rate.data(), prob.data(), len.data(), n);
    }
    if (!in->pendingOps.empty()) {
        std::vector<HostOp> hops;
        hops.swap(in->pendingOps);
        const int rc2 = planAndLaunch(in, hops, false);
        if (rc == BEAGLE_SUCCESS) rc = rc2;
    }
    return rc;
}

bool fusionPossible(const Instance* in) {
    return in->fuseSmall && in->matCP > 0 && in->matCP <= 8 && !in->timing && !in->exchangeOn && in->walkVariant == 0 &&
           in->eigenWalk && in->hMapped != nullptr;
}

// the whole deferred evaluation as one launch; the caller has checked eligibility
int launchFused(Instance* in, int E, int wIdx, int fIdx, int cum, double* outSum) {
    IncArgs A;
    memset(&A, 0, sizeof A);
    A.partials = in->partialsBase; A.stride = in->partialsElems; A.states = in->states8Base; A.mats = in->dMat;
    A.evecs = in->dEvec; A.scale = in->dScale; A.matStride = in->matStride;
    A.S = in->S; A.C = in->C; A.Ppad = in->Ppad; A.P = in->P; A.logScalers = in->logScalers ? 1 : 0;
    const double* h = in->hEigen.data() + (size_t)E * 36;
    for (int q = 0; q < 16; ++q) { A.V[q] = h[q]; A.Vi[q] = h[16 + q]; }
    for (int q = 0; q < 4; ++q) A.eval[q] = h[32 + q];
    A.nMats = (int)in->pendingMats.size();
    std::unordered_map<int, int> pendingOf;
    for (int q = 0; q < A.nMats; ++q) {
        A.mat[q] = IncMat{in->pendingMats[q].prob, in->pendingMats[q].rateSet, in->pendingMats[q].len};
        for (int c = 0; c < 8; ++c) A.rate[q][c] = c < in->C ? in->hRates[(size_t)in->pendingMats[q].rateSet * in->C + c] : 0.0;
        pendingOf[in->pendingMats[q].prob] = q;
    }
    A.nOps = (int)in->pendingOps.size();
    {
        // k_incremental reads stored partials only: every child not written by an EARLIER op of the list
        std::vector<int> outside;
        for (int k = 0; k < A.nOps; ++k)
            for (int c : {in->pendingOps[k].c1, in->pendingOps[k].c2}) {
                bool written = false;
                for (int w = 0; w < k; ++w) written = written || in->pendingOps[w].dest == c;
                if (!written) outside.push_back(c);
            }
        CUDA_OK(storeCherries(in, outside.data(), (int)outside.size()));
    }
    int prevDest = -1;
    for (int k = 0; k < A.nOps; ++k) {
        const HostOp& o = in->pendingOps[k];
        IncOp& d = A.op[k];
        const bool t1 = in->states32[o.c1] != nullptr, t2 = in->states32[o.c2] != nullptr;
        int c1 = o.c1, c2 = o.c2, m1 = o.m1, m2 = o.m2;
        d.flags = 0;
        if (k > 0 && !t1 && c1 == prevDest) d.flags = 1;
        else if (k > 0 && !t2 && c2 == prevDest) { std::swap(c1, c2); std::swap(m1, m2); d.flags = 1; }
        const bool s1 = in->states32[c1] != nullptr, s2 = in->states32[c2] != nullptr;
        d.dest = in->slotOf[o.dest];
        d.c1 = s1 ? -(c1 + 1) : in->slotOf[c1];
        d.c2 = s2 ? -(c2 + 1) : in->slotOf[c2];
        auto mat = [&](int m) { auto it = pendingOf.find(m); return it == pendingOf.end() ? m : -(it->second + 1); };
        d.m1 = mat(m1); d.m2 = mat(m2);
        d.sw = o.sw; d.sr = o.sw >= 0 ? -1 : o.sr;
        prevDest = o.dest;
    }
    for (int c = 0; c < 8; ++c) A.weights[c] = c < in->C ? in->hWeights[(size_t)wIdx * in->C + c] : 0.0;
    for (int i = 0; i < 4; ++i) A.freqs[i] = in->hFreqs[(size_t)fIdx * 4 + i];
    A.cum = cum == BEAGLE_OP_NONE ? nullptr : in->dScale + (size_t)cum * in->Ppad;
    A.patternWeights = in->dPatternWeights; A.site = in->dSite; A.blockSums = in->dIncSums; A.counter = in->dIncCounter;
    A.out = in->dOut;
    A.hostOut = in->dMapped;
    A.hostFlag = reinterpret_cast<volatile unsigned long long*>(in->dMapped + 1);
    A.seq = ++in->incSeq;
    CUDA_OK(launchIncremental(in, A));
    noteScaleWrites(in, in->pendingOps);
    noteCherryWrites(in, in->pendingOps, {});
    in->pendingMats.clear();
    in->pendingOps.clear();
    in->fusedLaunches++;
    // the result lands in mapped pinned memory: spin on the flag (bounded), no memcpy, no stream synchronise
    volatile unsigned long long* flag = reinterpret_cast<volatile unsigned long long*>(in->hMapped + 1);
    const auto t0 = std::chrono::steady_clock::now();
    long spins = 0;
    while (*flag != A.seq) {
        if ((++spins & 0xfff) == 0 &&
            std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > 5.0) {
            CUDA_OK(cudaStreamSynchronize(in->stream));       // a wedged device surfaces as an error here
            if (*flag != A.seq) return BEAGLE_ERROR_GENERAL;
        }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    *outSum = in->hMapped[0];
    return std::isnan(*outSum) ? BEAGLE_ERROR_FLOATING_POINT : BEAGLE_SUCCESS;
}
int flushPending(Instance* in) { return flushPendingImpl(in); }
}  // namespace
extern "C" {

int beagleUpdateTransitionMatrices(int instance, int eigenIndex, const int* probabilityIndices,
                                   const int* firstDerivativeIndices, const int* secondDerivativeIndices,
                                   const double* edgeLengths, int count) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleUpdateTransitionMatrices(c, eigenIndex, probabilityIndices, firstDerivativeIndices, secondDerivativeIndices, edgeLengths, count); }));
    GET_INSTANCE_LAZY(in, instance);
    if (firstDerivativeIndices != nullptr || secondDerivativeIndices != nullptr)
        return BEAGLE_ERROR_NO_IMPLEMENTATION;      // derivative matrices: SURVEY.md 8f "next"
    // a few branches of a real eigen system, nothing else pending: keep them for the one-launch evaluation (incr.cu)
    bool defer = fusionPossible(in) && count >= 1 && in->pendingOps.empty() &&
                 (int)in->pendingMats.size() + count <= kIncMaxMats && validRange(eigenIndex, in->nEigen) &&
                 in->eigenReal[eigenIndex] && in->eigenGen[eigenIndex] > 0;
    for (int k = 0; k < count && defer; ++k) {
        defer = validRange(probabilityIndices[k], in->nMatrices);
        for (const Instance::PendingMat& pm : in->pendingMats) defer = defer && pm.prob != probabilityIndices[k] && pm.eigen == eigenIndex;
        for (int q = 0; q < k && defer; ++q) defer = probabilityIndices[q] != probabilityIndices[k];
    }
    if (defer) {
        for (int k = 0; k < count; ++k) {
            in->pendingMats.push_back(Instance::PendingMat{probabilityIndices[k], eigenIndex, 0, edgeLengths[k]});
            in->matEigen[probabilityIndices[k]] = eigenIndex;
            in->matEigenGen[probabilityIndices[k]] = in->eigenGen[eigenIndex];
        }
        return BEAGLE_SUCCESS;
    }
    if (!in->pendingMats.empty() || !in->pendingOps.empty()) { const int rc = flushPending(in); if (rc != BEAGLE_SUCCESS) return rc; }
    return updateMatricesImpl(in, nullptr, eigenIndex, nullptr, probabilityIndices, edgeLengths, count);
}

int beagleUpdateTransitionMatricesWithMultipleModels(int instance, const int* eigenIndices,
                                                     const int* categoryRateIndices, const int* probabilityIndices,
                                                     const int* firstDerivativeIndices,
                                                     const int* secondDerivativeIndices, const double* edgeLengths,
                                                     int count) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleUpdateTransitionMatricesWithMultipleModels(c, eigenIndices, categoryRateIndices, probabilityIndices, firstDerivativeIndices, secondDerivativeIndices, edgeLengths, count); }));
    GET_INSTANCE(in, instance);
    if (firstDerivativeIndices != nullptr || secondDerivativeIndices != nullptr)
        return BEAGLE_ERROR_NO_IMPLEMENTATION;
    return updateMatricesImpl(in, eigenIndices, 0, categoryRateIndices, probabilityIndices, edgeLengths, count);
}

// device index of P[c][i][j] inside one matrix buffer (transposed; 4-state path: [j][CP][i])
static inline size_t matIndex(const Instance* in, int c, int i, int j) {
    return in->matCP ? ((size_t)j * in->matCP + c) * 4 + i : ((size_t)c * in->Sp + j) * in->Sp + i;
}

int beagleSetTransitionMatrix(int instance, int matrixIndex, const double* inMatrix, double) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleSetTransitionMatrix(c, matrixIndex, inMatrix, 0.0); }));
    GET_INSTANCE(in, instance);
    if (!validRange(matrixIndex, in->nMatrices)) return BEAGLE_ERROR_OUT_OF_RANGE;
    if (in->matCP > 0) in->matEigen[matrixIndex] = -1;        // set directly: no spectrum, matrix-form kernel only
    const size_t n = in->matStride;
    std::vector<double> t(n, 0.0);
    for (int c = 0; c < in->C; ++c)
        for (int i = 0; i < in->S; ++i)
            for (int j = 0; j < in->S; ++j)
            {
                const double v = inMatrix[((size_t)c * in->S + i) * in->S + j];
                t[matIndex(in, c, i, j)] = v;
                if (in->matCP) {
                    double* mm = t.data() + 16 * in->matCP;
                    mm[(size_t)c * 32 + i * 4 + j] = v;
                    double* mt = mm + (size_t)in->C * 32;
                    mt[(size_t)c * 20 + j * 4 + i] = v;
                    for (int q = 0; q < 4; ++q) {
                        if (in->S < 4) mt[(size_t)c * 20 + in->S * 4 + q] = q < in->S ? 1.0 : 0.0;
                        else mt[(size_t)c * 20 + 16 + q] = 1.0;
                    }
                } else {
                    const size_t ld = (size_t)in->Sp + 4, half = (size_t)in->C * in->Sp * in->Sp;
                    t[half + ((size_t)c * in->Sp + i) * ld + j] = v;
                    t[half + (size_t)in->C * in->Sp * ld + ((size_t)c * in->Sp + j) * ld + i] = v;
                }
            }
    CUDA_OK(cudaMemcpyAsync(in->dMat + matrixIndex * n, t.data(), sizeof(double) * n, cudaMemcpyHostToDevice, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    return BEAGLE_SUCCESS;
}

int beagleGetTransitionMatrix(int instance, int matrixIndex, double* outMatrix) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleGetTransitionMatrix(c, matrixIndex, outMatrix); }));
    GET_INSTANCE(in, instance);
    if (!validRange(matrixIndex, in->nMatrices)) return BEAGLE_ERROR_OUT_OF_RANGE;
    const size_t n = in->matStride;
    std::vector<double> t(n);
    CUDA_OK(cudaMemcpyAsync(t.data(), in->dMat + matrixIndex * n, sizeof(double) * n, cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    for (int c = 0; c < in->C; ++c)
        for (int i = 0; i < in->S; ++i)
            for (int j = 0; j < in->S; ++j)
                outMatrix[((size_t)c * in->S + i) * in->S + j] = t[matIndex(in, c, i, j)];
    return BEAGLE_SUCCESS;
}

int beagleSetDifferentialMatrix(int instance, int matrixIndex, const double* inMatrix) {
    return beagleSetTransitionMatrix(instance, matrixIndex, inMatrix, 0.0);     // same storage, all layouts
}
// SubstitutionModelDelegate.java:303-470 (epoch / branch-specific models): result = first x second per category,
// resp. first + second.  A handful of S x S products per call: done on the host between a get and a set.
static int combineMatrices(int instance, const int* firstIndices, const int* secondIndices, const int* resultIndices,
                           int matrixCount, bool multiply) {
    GET_INSTANCE(in, instance);
    if (matrixCount <= 0) return BEAGLE_SUCCESS;
    bool alias = false;
    for (int q = 0; q < matrixCount; ++q) {
        if (!validRange(firstIndices[q], in->nMatrices) || !validRange(secondIndices[q], in->nMatrices) ||
            !validRange(resultIndices[q], in->nMatrices))
            return BEAGLE_ERROR_OUT_OF_RANGE;
        for (int r2 = 0; r2 < matrixCount; ++r2)        // a result read (again) by any pair of the batch: ordered host path
            alias = alias || resultIndices[q] == firstIndices[r2] || resultIndices[q] == secondIndices[r2];
    }
    if (!alias) {
        // on the device: one launch for the whole batch (grid = pairs x categories), indices through the staging ring
        std::vector<int> idx(3 * (size_t)matrixCount);
        for (int q = 0; q < matrixCount; ++q) {
            idx[q] = firstIndices[q]; idx[matrixCount + q] = secondIndices[q]; idx[2 * (size_t)matrixCount + q] = resultIndices[q];
            if (in->matCP > 0) in->matEigen[resultIndices[q]] = -1;       // no spectrum: the matrix-form walk serves lists using it
        }
        int* d = static_cast<int*>(stage(in, idx.data(), sizeof(int) * idx.size()));
        if (d == nullptr) return BEAGLE_ERROR_OUT_OF_MEMORY;
        TimedScope ts(in, T_MATRICES);
        CUDA_OK(launchCombineMatrices(in, d, d + matrixCount, d + 2 * (size_t)matrixCount, matrixCount, multiply));
        return BEAGLE_SUCCESS;
    }
    const size_t n = (size_t)in->C * in->S * in->S;
    std::vector<double> a(n), b(n), r(n);
    for (int q = 0; q < matrixCount; ++q) {
        int rc = beagleGetTransitionMatrix(instance, firstIndices[q], a.data());
        if (rc == BEAGLE_SUCCESS) rc = beagleGetTransitionMatrix(instance, secondIndices[q], b.data());
        if (rc != BEAGLE_SUCCESS) return rc;
        const int S = in->S;
        for (int c = 0; c < in->C; ++c) {
            const double* A = a.data() + (size_t)c * S * S;
            const double* B = b.data() + (size_t)c * S * S;
            double* R = r.data() + (size_t)c * S * S;
            for (int i = 0; i < S; ++i)
                for (int j = 0; j < S; ++j) {
                    double v = 0.0;
                    if (multiply) for (int k = 0; k < S; ++k) v += A[i * S + k] * B[k * S + j];
                    else v = A[i * S + j] + B[i * S + j];
                    R[i * S + j] = v;
                }
        }
        rc = beagleSetTransitionMatrix(instance, resultIndices[q], r.data(), 0.0);
        if (rc != BEAGLE_SUCCESS) return rc;
    }
    return BEAGLE_SUCCESS;
}

int beagleConvolveTransitionMatrices(int instance, const int* firstIndices, const int* secondIndices,
                                     const int* resultIndices, int matrixCount) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleConvolveTransitionMatrices(c, firstIndices, secondIndices, resultIndices, matrixCount); }));
    return combineMatrices(instance, firstIndices, secondIndices, resultIndices, matrixCount, true);
}

int beagleAddTransitionMatrices(int instance, const int* firstIndices, const int* secondIndices, const int* resultIndices,
                                int matrixCount) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleAddTransitionMatrices(c, firstIndices, secondIndices, resultIndices, matrixCount); }));
    return combineMatrices(instance, firstIndices, secondIndices, resultIndices, matrixCount, false);
}
int beagleTransposeTransitionMatrices(int instance, const int* inputIndices, const int* resultIndices, int matrixCount) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleTransposeTransitionMatrices(c, inputIndices, resultIndices, matrixCount); }));
    GET_INSTANCE(in, instance);
    std::vector<double> m((size_t)in->C * in->S * in->S), t(m.size());
    for (int q = 0; q < matrixCount; ++q) {
        int rc = beagleGetTransitionMatrix(instance, inputIndices[q], m.data());
        if (rc != BEAGLE_SUCCESS) return rc;
        for (int c = 0; c < in->C; ++c)
            for (int i = 0; i < in->S; ++i)
                for (int j = 0; j < in->S; ++j)
                    t[((size_t)c * in->S + j) * in->S + i] = m[((size_t)c * in->S + i) * in->S + j];
        rc = beagleSetTransitionMatrix(instance, resultIndices[q], t.data(), 0.0);
        if (rc != BEAGLE_SUCCESS) return rc;
    }
    return BEAGLE_SUCCESS;
}

// ---- partials ---------------------------------------------------------------------------------
int beagleUpdatePartials(int instance, const BeagleOperation* operations, int operationCount,
                         int cumulativeScaleIndex) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleUpdatePartials(c, operations, operationCount, cumulativeScaleIndex); }));
    GET_INSTANCE_LAZY(in, instance);
    if (operationCount < 0) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<HostOp> hops(operationCount);
    for (int k = 0; k < operationCount; ++k) {
        const BeagleOperation& o = operations[k];
        hops[k] = {o.destinationPartials, o.destinationScaleWrite, o.destinationScaleRead, o.child1Partials,
                   o.child1TransitionMatrix, o.child2Partials, o.child2TransitionMatrix, 0, cumulativeScaleIndex};
    }
    // a short list in eigen form: hold it back, calculateRootLogLikelihoods will run matrices + list + root as ONE launch
    if (fusionPossible(in) && operationCount >= 1 && operationCount <= kIncMaxOps && in->pendingOps.empty() &&
        cumulativeScaleIndex == BEAGLE_OP_NONE) {
        bool ok = true;
        for (const HostOp& o : hops)
            ok = ok && validRange(o.m1, in->nMatrices) && validRange(o.m2, in->nMatrices);
        // The one-launch route runs the list as ONE dependent chain per pattern: right for what a move leaves dirty (one or two
        // root paths: every op consumes its predecessor's result), wrong for a short list with subtree parallelism (the whole
        // evaluation of a 62-taxon tree is 61 ops: the planned subtree walks finish it in a third of the time)
        int breaks = 0;
        for (int k = 1; k < operationCount; ++k)
            breaks += hops[k].c1 != hops[k - 1].dest && hops[k].c2 != hops[k - 1].dest;
        ok = ok && (breaks <= 2 || operationCount <= 16);
        const int E = ok ? eigenFormSlot(in, hops) : -1;
        for (const Instance::PendingMat& pm : in->pendingMats) ok = ok && pm.eigen == E;
        if (ok && E >= 0) {
            const int rc = prepareOps(in, hops, false);
            if (rc != BEAGLE_SUCCESS) return rc;
            in->pendingOps = hops;
            return BEAGLE_SUCCESS;
        }
    }
    if (!in->pendingMats.empty() || !in->pendingOps.empty()) { const int rc = flushPending(in); if (rc != BEAGLE_SUCCESS) return rc; }
    return planAndLaunch(in, hops, false);
}

int beagleUpdatePartialsByPartition(int instance, const BeagleOperationByPartition* operations, int operationCount) {
    SH(instance, BEAGLE_ERROR_NO_IMPLEMENTATION);
    GET_INSTANCE(in, instance);
    if (operationCount < 0) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<HostOp> hops(operationCount);
    for (int k = 0; k < operationCount; ++k) {
        const BeagleOperationByPartition& o = operations[k];
        hops[k] = {o.destinationPartials, o.destinationScaleWrite, o.destinationScaleRead, o.child1Partials,
                   o.child1TransitionMatrix, o.child2Partials, o.child2TransitionMatrix, o.partition,
                   o.cumulativeScaleIndex};
    }
    return planAndLaunch(in, hops, true);
}

int beagleWaitForPartials(int instance, const int*, int) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleWaitForPartials(c, nullptr, 0); }));
    GET_INSTANCE(in, instance);
    CUDA_OK(cudaStreamSynchronize(in->stream));
    return BEAGLE_SUCCESS;
}

int beagleUpdatePrePartials(int instance, const BeagleOperation* operations, int operationCount, int cumulativeScaleIndex) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleUpdatePrePartials(c, operations, operationCount, cumulativeScaleIndex); }));
    GET_INSTANCE(in, instance);
    if (operationCount < 0) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<HostOp> hops(operationCount);
    for (int k = 0; k < operationCount; ++k) {
        const BeagleOperation& o = operations[k];
        hops[k] = {o.destinationPartials, o.destinationScaleWrite, o.destinationScaleRead, o.child1Partials,
                   o.child1TransitionMatrix, o.child2Partials, o.child2TransitionMatrix, 0, cumulativeScaleIndex};
        hops[k].kind = 1;
    }
    return planAndLaunch(in, hops, false);
}
int beagleUpdatePrePartialsByPartition(int instance, const BeagleOperationByPartition* operations, int operationCount) {
    SH(instance, BEAGLE_ERROR_NO_IMPLEMENTATION);
    GET_INSTANCE(in, instance);
    if (operationCount < 0) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<HostOp> hops(operationCount);
    for (int k = 0; k < operationCount; ++k) {
        const BeagleOperationByPartition& o = operations[k];
        hops[k] = {o.destinationPartials, o.destinationScaleWrite, o.destinationScaleRead, o.child1Partials,
                   o.child1TransitionMatrix, o.child2Partials, o.child2TransitionMatrix, o.partition,
                   o.cumulativeScaleIndex};
        hops[k].kind = 1;
    }
    return planAndLaunch(in, hops, true);
}

// ---- scale factors ----------------------------------------------------------------------------
static int accumulateImpl(Instance* in, const int* scaleIndices, int count, int cum, double sign, int pBegin, int pEnd) {
    if (!validRange(cum, in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
    if (count <= 0) return BEAGLE_SUCCESS;
    for (int k = 0; k < count; ++k) if (!validRange(scaleIndices[k], in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
    int* dIdx = static_cast<int*>(stage(in, scaleIndices, sizeof(int) * count));
    if (dIdx == nullptr) return BEAGLE_ERROR_OUT_OF_MEMORY;
    TimedScope ts(in, T_ROOT);
    CUDA_OK(launchScaleAccumulate(in, dIdx, count, in->dScale + (size_t)cum * in->Ppad, sign, pBegin, pEnd));
    in->scaleIsLog[cum] = 1;
    return BEAGLE_SUCCESS;
}

int beagleAccumulateScaleFactors(int instance, const int* scaleIndices, int count, int cumulativeScaleIndex) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleAccumulateScaleFactors(c, scaleIndices, count, cumulativeScaleIndex); }));
    GET_INSTANCE(in, instance);
    return accumulateImpl(in, scaleIndices, count, cumulativeScaleIndex, 1.0, 0, in->P);
}

int beagleAccumulateScaleFactorsByPartition(int instance, const int* scaleIndices, int count,
                                            int cumulativeScaleIndex, int partitionIndex) {
    SH(instance, BEAGLE_ERROR_NO_IMPLEMENTATION);
    GET_INSTANCE(in, instance);
    if (!validRange(partitionIndex, in->partitionCount)) return BEAGLE_ERROR_OUT_OF_RANGE;
    return accumulateImpl(in, scaleIndices, count, cumulativeScaleIndex, 1.0, in->partBegin[partitionIndex],
                          in->partEnd[partitionIndex]);
}

int beagleRemoveScaleFactors(int instance, const int* scaleIndices, int count, int cumulativeScaleIndex) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleRemoveScaleFactors(c, scaleIndices, count, cumulativeScaleIndex); }));
    GET_INSTANCE(in, instance);
    return accumulateImpl(in, scaleIndices, count, cumulativeScaleIndex, -1.0, 0, in->P);
}

int beagleRemoveScaleFactorsByPartition(int instance, const int* scaleIndices, int count, int cumulativeScaleIndex,
                                        int partitionIndex) {
    SH(instance, BEAGLE_ERROR_NO_IMPLEMENTATION);
    GET_INSTANCE(in, instance);
    if (!validRange(partitionIndex, in->partitionCount)) return BEAGLE_ERROR_OUT_OF_RANGE;
    return accumulateImpl(in, scaleIndices, count, cumulativeScaleIndex, -1.0, in->partBegin[partitionIndex],
                          in->partEnd[partitionIndex]);
}

int beagleResetScaleFactors(int instance, int cumulativeScaleIndex) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleResetScaleFactors(c, cumulativeScaleIndex); }));
    GET_INSTANCE(in, instance);
    if (!validRange(cumulativeScaleIndex, in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(cudaMemsetAsync(in->dScale + (size_t)cumulativeScaleIndex * in->Ppad, 0, sizeof(double) * in->Ppad, in->stream));
    in->scaleIsLog[cumulativeScaleIndex] = 1;      // a cumulative buffer: sums of logs from here on
    return BEAGLE_SUCCESS;
}

int beagleResetScaleFactorsByPartition(int instance, int cumulativeScaleIndex, int partitionIndex) {
    SH(instance, BEAGLE_ERROR_NO_IMPLEMENTATION);
    GET_INSTANCE(in, instance);
    if (!validRange(cumulativeScaleIndex, in->nScale) || !validRange(partitionIndex, in->partitionCount))
        return BEAGLE_ERROR_OUT_OF_RANGE;
    int b = in->partBegin[partitionIndex], e = in->partEnd[partitionIndex];
    if (e > b)
        CUDA_OK(cudaMemsetAsync(in->dScale + (size_t)cumulativeScaleIndex * in->Ppad + b, 0, sizeof(double) * (e - b), in->stream));
    in->scaleIsLog[cumulativeScaleIndex] = 1;
    return BEAGLE_SUCCESS;
}

int beagleCopyScaleFactors(int instance, int destScalingIndex, int srcScalingIndex) {
    SH(instance, shBroadcast(sh, [&](int c) { return beagleCopyScaleFactors(c, destScalingIndex, srcScalingIndex); }));
    GET_INSTANCE(in, instance);
    if (!validRange(destScalingIndex, in->nScale) || !validRange(srcScalingIndex, in->nScale))
        return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(cudaMemcpyAsync(in->dScale + (size_t)destScalingIndex * in->Ppad, in->dScale + (size_t)srcScalingIndex * in->Ppad,
                            sizeof(double) * in->Ppad, cudaMemcpyDeviceToDevice, in->stream));
    in->scaleIsLog[destScalingIndex] = in->scaleIsLog[srcScalingIndex];
    return BEAGLE_SUCCESS;
}

int beagleGetScaleFactors(int instance, int srcScalingIndex, double* outScaleFactors) {
    SH(instance, shGetPerPattern(sh, outScaleFactors, [&](int c, double* o) { return beagleGetScaleFactors(c, srcScalingIndex, o); }));
    GET_INSTANCE(in, instance);
    if (!validRange(srcScalingIndex, in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(cudaMemcpyAsync(outScaleFactors, in->dScale + (size_t)srcScalingIndex * in->Ppad, sizeof(double) * in->P,
                            cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    return BEAGLE_SUCCESS;
}

int beagleGetLogScaleFactors(int instance, int srcScalingIndex, double* outLogScaleFactors) {
    SH(instance, shGetPerPattern(sh, outLogScaleFactors, [&](int c, double* o) { return beagleGetLogScaleFactors(c, srcScalingIndex, o); }));
    int rc = beagleGetScaleFactors(instance, srcScalingIndex, outLogScaleFactors);
    if (rc != BEAGLE_SUCCESS) return rc;
    Instance* in = getInstance(instance);
    // per-node buffers hold raw factors under SCALERS_RAW; cumulative buffers (reset / accumulate / in-list) always hold logs
    if (!in->scaleIsLog[srcScalingIndex])
        for (int p = 0; p < in->P; ++p) outLogScaleFactors[p] = log(outLogScaleFactors[p]);
    return BEAGLE_SUCCESS;
}

// ---- root -------------------------------------------------------------------------------------
static int rootLaunch(Instance* in, int buffer, int wIdx, int fIdx, int cum, int pBegin, int pEnd, double* dOutSlot,
                      bool joint = false) {
    if (!validRange(buffer, in->nBuffers) || in->partials[buffer] == nullptr || !validRange(wIdx, in->nSets) ||
        !validRange(fIdx, in->nSets))
        return BEAGLE_ERROR_OUT_OF_RANGE;
    if (cum != BEAGLE_OP_NONE && !validRange(cum, in->nScale)) return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(storeCherries(in, &buffer, 1));
    TimedScope ts(in, T_ROOT);
    const Exchange* ex = nullptr;
    if (joint && in->exchangeOn) {          // member of a reduce group: the kernel adds the other shards' sums (Exchange)
        in->exchange.seq++;
        ex = &in->exchange;
    }
    CUDA_OK(launchRoot(in, in->partials[buffer], in->dWeights + (size_t)wIdx * in->C, in->dFreqs + (size_t)fIdx * in->Sp,
                       cum == BEAGLE_OP_NONE ? nullptr : in->dScale + (size_t)cum * in->Ppad, pBegin, pEnd, dOutSlot, ex));
    return BEAGLE_SUCCESS;
}

int beagleCalculateRootLogLikelihoods(int instance, const int* bufferIndices, const int* categoryWeightsIndices,
                                      const int* stateFrequenciesIndices, const int* cumulativeScaleIndices,
                                      int count, double* outSumLogLikelihood) {
    SH(instance, shRoot(sh, bufferIndices, categoryWeightsIndices, stateFrequenciesIndices, cumulativeScaleIndices, count, outSumLogLikelihood));
    GET_INSTANCE_LAZY(in, instance);
    if (!in->pendingOps.empty() && count == 1 && fusionPossible(in) && bufferIndices[0] == in->pendingOps.back().dest &&
        validRange(categoryWeightsIndices[0], in->nSets) && validRange(stateFrequenciesIndices[0], in->nSets) &&
        (cumulativeScaleIndices[0] == BEAGLE_OP_NONE || validRange(cumulativeScaleIndices[0], in->nScale))) {
        const int E = eigenFormSlot(in, in->pendingOps);
        if (E >= 0)
            return launchFused(in, E, categoryWeightsIndices[0], stateFrequenciesIndices[0], cumulativeScaleIndices[0],
                               outSumLogLikelihood);
    }
    if (!in->pendingMats.empty() || !in->pendingOps.empty()) { const int rc = flushPending(in); if (rc != BEAGLE_SUCCESS) return rc; }
    if (count != 1) return BEAGLE_ERROR_NO_IMPLEMENTATION;   // BEAST always passes 1 (BDLD:934-935)
    int rc = rootLaunch(in, bufferIndices[0], categoryWeightsIndices[0], stateFrequenciesIndices[0],
                        cumulativeScaleIndices[0], 0, in->P, in->dOut, true);
    if (rc != BEAGLE_SUCCESS) return rc;
    CUDA_OK(cudaMemcpyAsync(in->hOut, in->dOut, sizeof(double), cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    *outSumLogLikelihood = in->hOut[0];
    return std::isnan(in->hOut[0]) ? BEAGLE_ERROR_FLOATING_POINT : BEAGLE_SUCCESS;
}

// launches of a *ByPartition root call: one k_root per listed partition into dOut[0..n); a member of a reduce group
// then adds the members' totals in one more tiny launch (dOut[n] = joint, dOut[n+1] = this member's total)
static int rootByPartitionLaunch(Instance* in, const int* bufferIndices, const int* categoryWeightsIndices,
                                 const int* stateFrequenciesIndices, const int* cumulativeScaleIndices,
                                 const int* partitionIndices, int partitionCount) {
    if (partitionCount < 1 || partitionCount > 1000) return BEAGLE_ERROR_OUT_OF_RANGE;
    for (int k = 0; k < partitionCount; ++k) {
        int part = partitionIndices[k];
        if (!validRange(part, in->partitionCount)) return BEAGLE_ERROR_OUT_OF_RANGE;
        int rc = rootLaunch(in, bufferIndices[k], categoryWeightsIndices[k], stateFrequenciesIndices[k],
                            cumulativeScaleIndices[k], in->partBegin[part], in->partEnd[part], in->dOut + k);
        if (rc != BEAGLE_SUCCESS) return rc;
    }
    if (in->exchangeOn) {
        in->exchange.seq++;
        TimedScope ts(in, T_ROOT);
        CUDA_OK(launchExchangeSum(in, in->dOut, partitionCount, in->dOut + partitionCount, &in->exchange));
    }
    return BEAGLE_SUCCESS;
}

int beagleCalculateRootLogLikelihoodsByPartition(int instance, const int* bufferIndices,
                                                 const int* categoryWeightsIndices,
                                                 const int* stateFrequenciesIndices,
                                                 const int* cumulativeScaleIndices, const int* partitionIndices,
                                                 int partitionCount, int count,
                                                 double* outSumLogLikelihoodByPartition, double* outSumLogLikelihood) {
    SH(instance, BEAGLE_ERROR_NO_IMPLEMENTATION);
    GET_INSTANCE(in, instance);
    if (count != 1) return BEAGLE_ERROR_NO_IMPLEMENTATION;
    int rc = rootByPartitionLaunch(in, bufferIndices, categoryWeightsIndices, stateFrequenciesIndices,
                                   cumulativeScaleIndices, partitionIndices, partitionCount);
    if (rc != BEAGLE_SUCCESS) return rc;
    const int extra = in->exchangeOn ? 2 : 0;
    CUDA_OK(cudaMemcpyAsync(in->hOut, in->dOut, sizeof(double) * (partitionCount + extra), cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    double total = 0.0;
    for (int k = 0; k < partitionCount; ++k) { outSumLogLikelihoodByPartition[k] = in->hOut[k]; total += in->hOut[k]; }
    if (in->exchangeOn) total = in->hOut[partitionCount];      // the sum over all members of the reduce group
    *outSumLogLikelihood = total;
    return std::isnan(total) ? BEAGLE_ERROR_FLOATING_POINT : BEAGLE_SUCCESS;
}

int beagleGetSiteLogLikelihoods(int instance, double* outLogLikelihoods) {
    SH(instance, shGetPerPattern(sh, outLogLikelihoods, [&](int c, double* o) { return beagleGetSiteLogLikelihoods(c, o); }));
    GET_INSTANCE(in, instance);
    CUDA_OK(cudaMemcpyAsync(outLogLikelihoods, in->dSite, sizeof(double) * in->P, cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    return BEAGLE_SUCCESS;
}

// ---- edge derivatives (pre-order route) ---------------------------------------------------------
// grow-only device workspace of the derivative calls (stream-ordered users only)
static cudaError_t ensureScratch(Instance* in, size_t doubles) {
    if (doubles <= in->scratchDoubles) return cudaSuccess;
    cudaError_t e = cudaStreamSynchronize(in->stream);
    if (e != cudaSuccess) return e;
    cudaFree(in->dScratch);
    in->dScratch = nullptr;
    in->scratchDoubles = 0;
    e = cudaMalloc(reinterpret_cast<void**>(&in->dScratch), doubles * sizeof(double));
    if (e == cudaSuccess) in->scratchDoubles = doubles;
    return e;
}

int beagleCalculateEdgeDerivatives(int instance, const int* postBufferIndices, const int* preBufferIndices,
                                   const int* derivativeMatrixIndices, const int* categoryWeightsIndices, int count,
                                   double* outDerivatives, double* outSumDerivatives, double* outSumSquaredDerivatives) {
    SH(instance, shEdgeDerivatives(sh, postBufferIndices, preBufferIndices, derivativeMatrixIndices, categoryWeightsIndices, count, outDerivatives, outSumDerivatives, outSumSquaredDerivatives));
    GET_INSTANCE(in, instance);
    if (count <= 0) return BEAGLE_SUCCESS;
    if (!validRange(categoryWeightsIndices[0], in->nSets)) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<EdgeRefT<void>> edges(count);
    for (int e = 0; e < count; ++e) {
        const int po = postBufferIndices[e], pr = preBufferIndices[e], dm = derivativeMatrixIndices[e];
        if (!validRange(po, in->nBuffers) || !validRange(pr, in->nBuffers) || !validRange(dm, in->nMatrices) ||
            in->partials[pr] == nullptr || (in->partials[po] == nullptr && in->states32[po] == nullptr))
            return BEAGLE_ERROR_OUT_OF_RANGE;
        edges[e].post = in->states32[po] != nullptr ? nullptr : in->partials[po];
        edges[e].states = in->states32[po];
        edges[e].pre = in->partials[pr];
        edges[e].D = in->dMat + (size_t)dm * in->matStride;
        edges[e].len = 0.0;
    }
    CUDA_OK(storeCherries(in, postBufferIndices, count));
    // workspace: [edge records][sum, sumSquared per edge][per-pattern values (optional)][tile partials (tensor form)]
    const size_t perEdge = outDerivatives != nullptr ? (size_t)in->P : 0;
    const size_t edgeDoubles = ((size_t)count * sizeof(EdgeRefT<void>) + 7) / 8;
    const size_t results = (size_t)count * (2 + perEdge);
    const size_t partials = edgeDerivativeWorkspace(in, count);
    CUDA_OK(ensureScratch(in, edgeDoubles + results + partials));
    EdgeRefT<void>* dEdges = reinterpret_cast<EdgeRefT<void>*>(in->dScratch);
    double* dOut = in->dScratch + edgeDoubles;
    CUDA_OK(cudaMemcpyAsync(dEdges, edges.data(), sizeof(EdgeRefT<void>) * count, cudaMemcpyHostToDevice, in->stream));
    {
        TimedScope ts(in, T_ROOT);
        CUDA_OK(launchEdgeDerivatives(in, dEdges, count, in->dWeights + (size_t)categoryWeightsIndices[0] * in->C,
                                      perEdge ? dOut + 2 * (size_t)count : nullptr, dOut, dOut + count,
                                      partials ? dOut + results : nullptr));
    }
    std::vector<double> host(results);
    CUDA_OK(cudaMemcpyAsync(host.data(), dOut, sizeof(double) * results, cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    for (int k = 0; k < count; ++k) {
        if (outSumDerivatives) outSumDerivatives[k] = host[k];
        if (outSumSquaredDerivatives) outSumSquaredDerivatives[k] = host[count + k];
    }
    if (outDerivatives) memcpy(outDerivatives, host.data() + 2 * (size_t)count, sizeof(double) * (size_t)count * in->P);
    return BEAGLE_SUCCESS;
}

// Beagle.calculateCrossProductDifferentials (SubstitutionModelCrossProductDelegate.java:158-176): S x S sums over the
// listed branches, ADDED to outSumDerivatives (the caller zero-fills it first, :156,:169).
int beagleCalculateCrossProductDerivative(int instance, const int* postBufferIndices, const int* preBufferIndices,
                                          const int* categoryRatesIndices, const int* categoryWeightsIndices,
                                          const double* edgeLengths, int count, double* outSumDerivatives,
                                          double* outSumSquaredDerivatives) {
    SH(instance, shCrossProducts(sh, postBufferIndices, preBufferIndices, categoryRatesIndices, categoryWeightsIndices, edgeLengths, count, outSumDerivatives, outSumSquaredDerivatives));
    GET_INSTANCE(in, instance);
    if (outSumSquaredDerivatives != nullptr) return BEAGLE_ERROR_NO_IMPLEMENTATION;   // BEAST passes null (:161,:175)
    if (count <= 0) return BEAGLE_SUCCESS;
    if (outSumDerivatives == nullptr || edgeLengths == nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
    if (!validRange(categoryRatesIndices[0], in->nSets) || !validRange(categoryWeightsIndices[0], in->nSets))
        return BEAGLE_ERROR_OUT_OF_RANGE;
    const size_t n = (size_t)in->S * in->S;
    const size_t edgeDoubles = ((size_t)count * sizeof(EdgeRefT<void>) + 7) / 8;
    const size_t need = edgeDoubles + ((size_t)crossProductBlocks(in, count) + 1) * n;
    CUDA_OK(ensureScratch(in, need));
    std::vector<EdgeRefT<void>> edges(count);
    for (int e = 0; e < count; ++e) {
        const int po = postBufferIndices[e], pr = preBufferIndices[e];
        if (!validRange(po, in->nBuffers) || !validRange(pr, in->nBuffers) || in->partials[pr] == nullptr ||
            (in->partials[po] == nullptr && in->states32[po] == nullptr))
            return BEAGLE_ERROR_OUT_OF_RANGE;
        edges[e].post = in->states32[po] != nullptr ? nullptr : in->partials[po];
        edges[e].states = in->states32[po];
        edges[e].pre = in->partials[pr];
        edges[e].D = nullptr;
        edges[e].len = edgeLengths[e];
    }
    CUDA_OK(storeCherries(in, postBufferIndices, count));
    EdgeRefT<void>* dEdges = reinterpret_cast<EdgeRefT<void>*>(in->dScratch);
    double* work = in->dScratch + edgeDoubles;
    CUDA_OK(cudaMemcpyAsync(dEdges, edges.data(), sizeof(EdgeRefT<void>) * count, cudaMemcpyHostToDevice, in->stream));
    {
        TimedScope ts(in, T_ROOT);
        CUDA_OK(launchCrossProducts(in, dEdges, count, in->dRates + (size_t)categoryRatesIndices[0] * in->C,
                                    in->dWeights + (size_t)categoryWeightsIndices[0] * in->C, work));
    }
    std::vector<double> host(n);
    CUDA_OK(cudaMemcpyAsync(host.data(), work + (size_t)crossProductBlocks(in, count) * n, sizeof(double) * n,
                            cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    for (size_t q = 0; q < n; ++q) outSumDerivatives[q] += host[q];
    return BEAGLE_SUCCESS;
}

// ---- host-logic test hook (no CUDA calls): the execution plan of an operation list -----------------
int b200DebugPlan(const int* operations, int operationCount, int bufferCount, int fixedT, int wantSubs, int minT,
                  int smallRemainder, int preOrder, int* outOrder, int* outSubs, int* outPhaseStart, int* outCounts) {
    if (operationCount < 0 || bufferCount <= 0) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<HostOp> hops(operationCount);
    for (int k = 0; k < operationCount; ++k) {
        const int* o = operations + 7 * k;
        for (int f : {o[0], o[3], o[5]}) if (f < 0 || f >= bufferCount) return BEAGLE_ERROR_OUT_OF_RANGE;
        hops[k] = {o[0], o[1], o[2], o[3], o[4], o[5], o[6], 0, -1};
        hops[k].kind = preOrder ? 1 : 0;
    }
    Plan plan;
    if (operationCount == 0) { outCounts[0] = outCounts[1] = 0; return BEAGLE_SUCCESS; }
    if (preOrder == 2) planLevels(hops, bufferCount, plan);
    else if (preOrder) planPreorderPhases(hops, bufferCount, fixedT, std::max(1, wantSubs), std::max(1, minT), smallRemainder, plan);
    else planPhases(hops, bufferCount, true, fixedT, std::max(1, wantSubs), std::max(1, minT), smallRemainder, plan);
    for (int k = 0; k < operationCount; ++k) outOrder[k] = plan.order[k];
    for (size_t q = 0; q < plan.subs.size(); ++q) { outSubs[2 * q] = plan.subs[q].begin; outSubs[2 * q + 1] = plan.subs[q].end; }
    for (size_t q = 0; q < plan.phaseStart.size(); ++q) outPhaseStart[q] = plan.phaseStart[q];
    outCounts[0] = (int)plan.subs.size();
    outCounts[1] = (int)plan.phaseStart.size() - 1;
    return BEAGLE_SUCCESS;
}

// ---- host-logic test hook (no CUDA calls): register forwarding and sibling-stack slots of a post-order list -----------
int b200DebugStackSlots(const int* operations, int operationCount, int bufferCount, int tipCount, int wantSubs, int minT,
                        int smallRemainder, int* outRecords, int* outSubs, int* outPhaseStart, int* outCounts) {
    if (operationCount <= 0 || bufferCount <= 0 || tipCount < 0 || tipCount > bufferCount) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::vector<HostOp> hops(operationCount);
    for (int k = 0; k < operationCount; ++k) {
        const int* o = operations + 7 * k;
        for (int f : {o[0], o[3], o[5]}) if (f < 0 || f >= bufferCount) return BEAGLE_ERROR_OUT_OF_RANGE;
        hops[k] = {o[0], o[1], o[2], o[3], o[4], o[5], o[6], 0, -1};
    }
    Plan plan;
    planPhases(hops, bufferCount, true, 0, std::max(1, wantSubs), std::max(1, minT), smallRemainder, plan);
    std::vector<Op4> ops(operationCount);
    for (int pos = 0; pos < operationCount; ++pos) {            // buffers below tipCount are compact tips
        const HostOp& o = hops[plan.order[pos]];
        Op4& d = ops[pos];
        memset(&d, 0, sizeof d);
        d.dest = o.dest;
        d.c1 = o.c1 < tipCount ? -(o.c1 + 1) : o.c1;
        d.c2 = o.c2 < tipCount ? -(o.c2 + 1) : o.c2;
        d.m1 = o.m1; d.m2 = o.m2; d.pEnd = 1;
        d.slots = 0xFFFFFFu;
    }
    for (size_t s = 0; s < plan.subs.size(); ++s)
        for (int pos = plan.subs[s].begin + 1; pos < plan.subs[s].end; ++pos) forwardFromPrevious(ops[pos], ops[pos - 1], false, nullptr);
    std::vector<int> subDepth;
    long fromStack = 0, fromMemory = 0;
    assignStackSlots(ops, plan.subs, kStackSlots, subDepth, fromStack, fromMemory);
    for (int pos = 0; pos < operationCount; ++pos) {
        const Op4& d = ops[pos];
        int* r = outRecords + 5 * pos;
        r[0] = d.dest; r[1] = d.c1; r[2] = d.c2; r[3] = d.pad_; r[4] = (int)d.slots;
    }
    for (size_t q = 0; q < plan.subs.size(); ++q) { outSubs[2 * q] = plan.subs[q].begin; outSubs[2 * q + 1] = plan.subs[q].end; }
    for (size_t q = 0; q < plan.phaseStart.size(); ++q) outPhaseStart[q] = plan.phaseStart[q];
    outCounts[0] = (int)plan.subs.size();
    outCounts[1] = (int)plan.phaseStart.size() - 1;
    outCounts[2] = (int)fromStack;
    outCounts[3] = (int)fromMemory;
    outCounts[4] = *std::max_element(subDepth.begin(), subDepth.end());
    return BEAGLE_SUCCESS;
}

// ---- joint ancestral-state sampling (ancestral.cu) ---------------------------------------------------------------------
// the row rules, no CUDA calls: row 0 is the root (parent -1; its node buffer and matrix are not read), every later row
// names a buffer, a parent row before it and a matrix buffer
int b200DebugAncestralRows(const int* nodeBuffers, const int* parentRows, const int* matrixIndices, int count,
                           int bufferCount, int matrixCount) {
    if (count < 1 || nodeBuffers == nullptr || parentRows == nullptr || matrixIndices == nullptr || parentRows[0] != -1)
        return BEAGLE_ERROR_OUT_OF_RANGE;
    for (int r = 1; r < count; ++r)
        if (!validRange(nodeBuffers[r], bufferCount) || !validRange(parentRows[r], r) || !validRange(matrixIndices[r], matrixCount))
            return BEAGLE_ERROR_OUT_OF_RANGE;
    return BEAGLE_SUCCESS;
}

int b200SampleAncestralStates(int instance, const int* nodeBuffers, const int* parentRows, const int* matrixIndices, int count,
                              int rootBuffer, int categoryWeightsIndex, int stateFrequenciesIndex, unsigned long long seed,
                              unsigned long long drawIndex, int* outStates, int* outCategories) {
    SH(instance, shSampleAncestralStates(sh, nodeBuffers, parentRows, matrixIndices, count, rootBuffer, categoryWeightsIndex,
                                         stateFrequenciesIndex, seed, drawIndex, outStates, outCategories));
    return sampleAncestralStates(instance, nodeBuffers, parentRows, matrixIndices, count, rootBuffer, categoryWeightsIndex,
                                 stateFrequenciesIndex, seed, drawIndex, 0, outStates, outCategories);
}

int b200SampleMarkovJumps(int instance, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                          const double* edgeLengths, int count, int rootBuffer, int categoryWeightsIndex,
                          int stateFrequenciesIndex, int eigenIndex, int categoryRatesIndex, const double* registerMatrices,
                          int registerCount, unsigned long long seed, unsigned long long drawIndex, int* outStates,
                          int* outCategories, double* outBranchCounts, double* outPatternCounts) {
    SH(instance, shSampleMarkovJumps(sh, nodeBuffers, parentRows, matrixIndices, edgeLengths, count, rootBuffer,
                                     categoryWeightsIndex, stateFrequenciesIndex, eigenIndex, categoryRatesIndex,
                                     registerMatrices, registerCount, seed, drawIndex, outStates, outCategories,
                                     outBranchCounts, outPatternCounts));
    return sampleMarkovJumps(instance, nodeBuffers, parentRows, matrixIndices, edgeLengths, count, rootBuffer,
                             categoryWeightsIndex, stateFrequenciesIndex, eigenIndex, categoryRatesIndex, registerMatrices,
                             registerCount, seed, drawIndex, 0, outStates, outCategories, outBranchCounts, outPatternCounts);
}

}  // extern "C"

// the sampler's argument rules and the written state of every buffer it reads: checked before anything is launched, the
// deferred work of earlier calls included
static int checkSampleRows(Instance* in, const int* nodeBuffers, const int* parentRows, const int* matrixIndices, int count,
                           int rootBuffer, int categoryWeightsIndex, int stateFrequenciesIndex) {
    if (b200DebugAncestralRows(nodeBuffers, parentRows, matrixIndices, count, in->nBuffers, in->nMatrices) != BEAGLE_SUCCESS ||
        !validRange(rootBuffer, in->nBuffers) || !validRange(categoryWeightsIndex, in->nSets) ||
        !validRange(stateFrequenciesIndex, in->nSets))
        return BEAGLE_ERROR_OUT_OF_RANGE;
    // a buffer must hold data: partials (a deferred list has already assigned its destinations) or compact states
    auto holdsData = [&](int b) { return in->partials[b] != nullptr || in->states32[b] != nullptr; };
    if (!holdsData(rootBuffer)) return BEAGLE_ERROR_OUT_OF_RANGE;
    for (int r = 1; r < count; ++r) if (!holdsData(nodeBuffers[r])) return BEAGLE_ERROR_OUT_OF_RANGE;
    return BEAGLE_SUCCESS;
}

// after checkSampleRows: flushes the deferred work, stores virtual cherries, grows the scratch to the sampler's int outputs
// [categories P | states count x P] followed by `extraDoubles` (*extra), stages the rows and fills the sampler's arguments
static int prepareSample(Instance* in, const int* nodeBuffers, const int* parentRows, const int* matrixIndices, int count,
                         int rootBuffer, int categoryWeightsIndex, int stateFrequenciesIndex, unsigned long long seed,
                         unsigned long long drawIndex, int patternOffset, size_t extraDoubles, AncestralArgs& a,
                         double** extra) {
    if (!in->pendingMats.empty() || !in->pendingOps.empty()) { const int rc = flushPending(in); if (rc != BEAGLE_SUCCESS) return rc; }
    std::vector<int> bufs(nodeBuffers, nodeBuffers + count);
    bufs[0] = rootBuffer;
    CUDA_OK(storeCherries(in, bufs.data(), count));       // virtual cherries have no stored partials until asked for them
    std::vector<int4> rows(count);
    for (int r = 0; r < count; ++r) {
        const int b = bufs[r];
        rows[r] = make_int4(in->states32[b] != nullptr ? -(b + 1) : in->slotOf[b], r == 0 ? -1 : parentRows[r],
                            r == 0 ? 0 : matrixIndices[r], 0);
    }
    const size_t intDoubles = ((size_t)(count + 1) * in->P + 1) / 2;
    CUDA_OK(ensureScratch(in, intDoubles + extraDoubles));
    const int4* dRows = static_cast<const int4*>(stage(in, rows.data(), sizeof(int4) * count));
    if (dRows == nullptr) return BEAGLE_ERROR_OUT_OF_MEMORY;
    a.rows = dRows; a.count = count; a.P = in->P; a.Ppad = in->Ppad; a.S = in->S; a.Sp = in->Sp; a.C = in->C; a.CP = in->matCP;
    a.pOffset = patternOffset;
    a.partials = in->partialsBase; a.stride = in->partialsElems;
    a.states8 = in->states8Base; a.states32 = in->states32Base;
    a.mats = in->dMat; a.matStride = in->matStride;
    a.weights = in->dWeights + (size_t)categoryWeightsIndex * in->C;
    a.freqs = in->dFreqs + (size_t)stateFrequenciesIndex * in->Sp;
    a.seed = seed; a.drawIndex = drawIndex;
    int* dOut = reinterpret_cast<int*>(in->dScratch);
    a.outCategories = dOut;
    a.outStates = dOut + in->P;
    if (extra != nullptr) *extra = in->dScratch + intDoubles;
    return BEAGLE_SUCCESS;
}

int b200::sampleAncestralStates(int instance, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                                int count, int rootBuffer, int categoryWeightsIndex, int stateFrequenciesIndex,
                                unsigned long long seed, unsigned long long drawIndex, int patternOffset, int* outStates,
                                int* outCategories) {
    GET_INSTANCE_LAZY(in, instance);
    if (outStates == nullptr || outCategories == nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
    int rc = checkSampleRows(in, nodeBuffers, parentRows, matrixIndices, count, rootBuffer, categoryWeightsIndex,
                             stateFrequenciesIndex);
    if (rc != BEAGLE_SUCCESS) return rc;
    AncestralArgs a;
    rc = prepareSample(in, nodeBuffers, parentRows, matrixIndices, count, rootBuffer, categoryWeightsIndex, stateFrequenciesIndex,
                       seed, drawIndex, patternOffset, 0, a, nullptr);
    if (rc != BEAGLE_SUCCESS) return rc;
    CUDA_OK(launchAncestral(in, a));
    const size_t outInts = (size_t)(count + 1) * in->P;          // [categories P | states count x P]: ONE D2H copy
    std::vector<int> host(outInts);
    CUDA_OK(cudaMemcpyAsync(host.data(), a.outCategories, sizeof(int) * outInts, cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    memcpy(outCategories, host.data(), sizeof(int) * in->P);
    memcpy(outStates, host.data() + in->P, sizeof(int) * (size_t)count * in->P);
    return BEAGLE_SUCCESS;
}

int b200::sampleMarkovJumps(int instance, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                            const double* edgeLengths, int count, int rootBuffer, int categoryWeightsIndex,
                            int stateFrequenciesIndex, int eigenIndex, int categoryRatesIndex, const double* registerMatrices,
                            int registerCount, unsigned long long seed, unsigned long long drawIndex, int patternOffset,
                            int* outStates, int* outCategories, double* outBranchCounts, double* outPatternCounts) {
    GET_INSTANCE_LAZY(in, instance);
    int rc = checkSampleRows(in, nodeBuffers, parentRows, matrixIndices, count, rootBuffer, categoryWeightsIndex,
                             stateFrequenciesIndex);
    if (rc != BEAGLE_SUCCESS) return rc;
    if (!validRange(eigenIndex, in->nEigen) || in->eigenKind[eigenIndex] == 0 || !validRange(categoryRatesIndex, in->nSets) ||
        edgeLengths == nullptr || registerMatrices == nullptr || registerCount < 1 || registerCount > kMaxJumpRegisters ||
        (outBranchCounts == nullptr && outPatternCounts == nullptr))
        return BEAGLE_ERROR_OUT_OF_RANGE;
    for (int r = 1; r < count; ++r)
        if (!(std::isfinite(edgeLengths[r]) && edgeLengths[r] >= 0.0)) return BEAGLE_ERROR_OUT_OF_RANGE;
    if (in->eigenKind[eigenIndex] != 1 || !markovJumpsFit(in)) return BEAGLE_ERROR_NO_IMPLEMENTATION;
    // scratch after the sampler's ints: M | W [G][S][S], N [G][count][C][S][S], pattern [G][P], branch [G][count] and, for
    // the branch totals only, the per-(row, pattern) workspace [G][count][P]
    const size_t G = registerCount, SS = (size_t)in->S * in->S, R = count, P = in->P;
    const size_t nCond = G * R * in->C * SS, nPerRow = outBranchCounts != nullptr ? G * R * P : 0;
    AncestralArgs a;
    double* x = nullptr;
    rc = prepareSample(in, nodeBuffers, parentRows, matrixIndices, count, rootBuffer, categoryWeightsIndex, stateFrequenciesIndex,
                       seed, drawIndex, patternOffset, 2 * G * SS + nCond + G * P + G * R + nPerRow, a, &x);
    if (rc != BEAGLE_SUCCESS) return rc;
    MarkovJumpArgs m;
    m.G = registerCount;
    m.eigen = in->dEigen + (size_t)eigenIndex * (2 * SS + 2 * in->S);
    m.rates = in->dRates + (size_t)categoryRatesIndex * in->C;
    double* dM = x;
    m.registers = dM;
    m.W = dM + G * SS;
    m.cond = m.W + G * SS;
    m.pattern = m.cond + nCond;
    m.branch = m.pattern + G * P;
    m.perRow = outBranchCounts != nullptr ? m.branch + G * R : nullptr;
    if (outBranchCounts == nullptr) m.branch = nullptr;
    m.patternWeights = in->dPatternWeights;
    rc = uploadSmall(in, dM, registerMatrices, sizeof(double) * G * SS);
    if (rc != BEAGLE_SUCCESS) return rc;
    m.lengths = static_cast<const double*>(stage(in, edgeLengths, sizeof(double) * R));
    if (m.lengths == nullptr) return BEAGLE_ERROR_OUT_OF_MEMORY;
    if (outPatternCounts == nullptr) m.pattern = nullptr;
    CUDA_OK(launchMarkovJumps(in, a, m));
    // only what was asked for comes back
    std::vector<int> ints(outStates != nullptr ? (size_t)(count + 1) * P : outCategories != nullptr ? P : 0);
    if (!ints.empty())
        CUDA_OK(cudaMemcpyAsync(ints.data(), a.outCategories, sizeof(int) * ints.size(), cudaMemcpyDeviceToHost, in->stream));
    if (outBranchCounts != nullptr)
        CUDA_OK(cudaMemcpyAsync(outBranchCounts, m.branch, sizeof(double) * G * R, cudaMemcpyDeviceToHost, in->stream));
    if (outPatternCounts != nullptr)
        CUDA_OK(cudaMemcpyAsync(outPatternCounts, m.pattern, sizeof(double) * G * P, cudaMemcpyDeviceToHost, in->stream));
    CUDA_OK(cudaStreamSynchronize(in->stream));
    if (outCategories != nullptr) memcpy(outCategories, ints.data(), sizeof(int) * P);
    if (outStates != nullptr) memcpy(outStates, ints.data() + P, sizeof(int) * R * P);
    return BEAGLE_SUCCESS;
}

extern "C" {

// ---- engine extensions ------------------------------------------------------------------------
int b200SetKernelTiming(int instance, int enable) {
    SH(instance, shBroadcast(sh, [&](int c) { return b200SetKernelTiming(c, enable); }));
    GET_INSTANCE(in, instance);
    CUDA_OK(cudaStreamSynchronize(in->stream));
    for (int c = 0; c < T_CLASSES; ++c) {
        for (auto& ev : in->timed[c]) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
        in->timed[c].clear();
        in->timedMs[c] = 0.0;
        in->timedLaunches[c] = 0;
    }
    in->timing = enable != 0;
    return BEAGLE_SUCCESS;
}

int b200GetKernelTiming(int instance, int which, double* outMilliseconds, long* outLaunches) {
    GET_INSTANCE(in, instance);
    if (which < 0 || which >= T_CLASSES) return BEAGLE_ERROR_OUT_OF_RANGE;
    CUDA_OK(cudaStreamSynchronize(in->stream));
    for (auto& ev : in->timed[which]) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) in->timedMs[which] += ms;
        in->timedLaunches[which]++;
        cudaEventDestroy(ev.first);
        cudaEventDestroy(ev.second);
    }
    in->timed[which].clear();
    if (outMilliseconds) *outMilliseconds = in->timedMs[which];
    if (outLaunches) *outLaunches = in->timedLaunches[which];
    return BEAGLE_SUCCESS;
}

int b200CompressSitePatterns(int resourceNumber, int taxonCount, int siteCount, const int* inStates,
                             const double* inSiteWeights, int* outSitePatternIndices, int* outPatterns,
                             double* outWeights, int* outPatternCount) {
    BeagleResourceList* rl = beagleGetResourceList();
    if (rl == nullptr || resourceNumber < 1 || resourceNumber >= rl->length) return BEAGLE_ERROR_NO_RESOURCE;
    if (taxonCount < 1 || taxonCount > 65535 || siteCount < 0 || outPatternCount == nullptr) return BEAGLE_ERROR_OUT_OF_RANGE;
    if (siteCount > 0 && (inStates == nullptr || outSitePatternIndices == nullptr || outPatterns == nullptr ||
                          outWeights == nullptr))
        return BEAGLE_ERROR_OUT_OF_RANGE;
    const int rc = compressSitePatterns(resourceNumber - 1, taxonCount, siteCount, inStates, outSitePatternIndices,
                                        outPatterns, outWeights, outPatternCount);
    if (rc != 0) return rc;
    if (inSiteWeights != nullptr) {
        // weights[i] += weight in site order, the order SitePatterns.addPattern adds them (:361-365)
        for (int p = 0; p < *outPatternCount; ++p) outWeights[p] = 0.0;
        for (int s = 0; s < siteCount; ++s) outWeights[outSitePatternIndices[s]] += inSiteWeights[s];
    }
    return BEAGLE_SUCCESS;
}

// -beagle_auto (BDLD:400-434): time a synthetic full evaluation of the stated shape on every candidate resource through
// the public entry points and return the resources fastest first.  Resource 0 (host) is not implemented and never listed.
BeagleBenchmarkedResourceList* beagleGetBenchmarkedResourceList(
    int tipCount, int compactBufferCount, int stateCount, int patternCount, int categoryCount, int* resourceList,
    int resourceCount, long preferenceFlags, long requirementFlags, int eigenModelCount, int partitionCount,
    int calculateDerivatives, long benchmarkFlags) {
    (void)eigenModelCount; (void)partitionCount; (void)calculateDerivatives; (void)compactBufferCount;
    static std::mutex mu;
    static std::vector<BeagleBenchmarkedResource> results;
    static BeagleBenchmarkedResourceList list;
    static const char* kImpl = "B200-CUDA-Double";
    std::lock_guard<std::mutex> lock(mu);
    BeagleResourceList* rl = beagleGetResourceList();
    if (rl == nullptr || tipCount < 2 || stateCount < 2 || patternCount < 1 || categoryCount < 1) return nullptr;
    std::vector<int> candidates;
    if (resourceList != nullptr && resourceCount > 0) {
        for (int k = 0; k < resourceCount; ++k)
            if (resourceList[k] >= 1 && resourceList[k] < rl->length &&
                std::find(candidates.begin(), candidates.end(), resourceList[k]) == candidates.end())
                candidates.push_back(resourceList[k]);
    } else {
        for (int r = 1; r < rl->length; ++r) candidates.push_back(r);
    }
    const bool rescale = (benchmarkFlags & 2L) != 0 || (benchmarkFlags & 4L) != 0;    // SCALING_ALWAYS / SCALING_DYNAMIC
    const int N = tipCount, n = 2 * N - 1, S = stateCount, P = patternCount, C = categoryCount;
    // synthetic inputs: pseudo-random tip states, a diagonal eigen system (P(t) = diag(exp(-k t / S))), a caterpillar tree
    std::vector<int> states(P);
    std::vector<double> evec((size_t)S * S, 0.0), eval(S), ones(std::max(std::max(C, S), P), 1.0), lengths(n - 1, 0.05);
    for (int i = 0; i < S; ++i) { evec[(size_t)i * S + i] = 1.0; eval[i] = -(double)i / S; }
    for (double& f : ones) f = 1.0;
    std::vector<double> freqs(S, 1.0 / S), weights(C, 1.0 / C), rates(C, 1.0);
    std::vector<int> probIdx(n - 1), ops, scaleIdx;
    for (int k = 0; k < n - 1; ++k) probIdx[k] = k;
    for (int k = 0; k < N - 1; ++k) {           // node N+k = (previous node or tip 0, tip k+1)
        const int dest = N + k, c1 = k == 0 ? 0 : N + k - 1, c2 = k + 1;
        const int sw = rescale ? k : BEAGLE_OP_NONE;
        const int tuple[7] = {dest, sw, BEAGLE_OP_NONE, c1, c1, c2, c2};
        ops.insert(ops.end(), tuple, tuple + 7);
        scaleIdx.push_back(k);
    }
    results.clear();
    for (int res : candidates) {
        BeagleBenchmarkedResource br{};
        br.number = res; br.name = rl->list[res].name; br.description = rl->list[res].description;
        br.supportFlags = rl->list[res].supportFlags; br.requiredFlags = rl->list[res].requiredFlags;
        br.implName = const_cast<char*>(kImpl); br.benchedFlags = 0; br.benchmarkResult = 0.0; br.performanceRatio = 0.0;
        int one[1] = {res};
        BeagleInstanceDetails det{};
        const int inst = beagleCreateInstance(N, N - 1, N, S, P, 1, n - 1, C, N + 1, one, 1, preferenceFlags,
                                              requirementFlags, &det);
        br.returnCode = inst < 0 ? inst : BEAGLE_SUCCESS;
        if (inst >= 0) {
            br.benchedFlags = det.flags;
            int rc = BEAGLE_SUCCESS;
            for (int t = 0; t < N && rc == BEAGLE_SUCCESS; ++t) {
                for (int p = 0; p < P; ++p) states[p] = (int)((1103515245u * (unsigned)(t * 7919 + p) + 12345u) >> 16) % S;
                rc = beagleSetTipStates(inst, t, states.data());
            }
            if (rc == BEAGLE_SUCCESS) rc = beagleSetPatternWeights(inst, ones.data());
            if (rc == BEAGLE_SUCCESS) rc = beagleSetEigenDecomposition(inst, 0, evec.data(), evec.data(), eval.data());
            if (rc == BEAGLE_SUCCESS) rc = beagleSetCategoryRates(inst, rates.data());
            if (rc == BEAGLE_SUCCESS) rc = beagleSetCategoryWeights(inst, 0, weights.data());
            if (rc == BEAGLE_SUCCESS) rc = beagleSetStateFrequencies(inst, 0, freqs.data());
            double best = 0.0, logL = 0.0;
            const int root = n - 1, zero = 0, cum = rescale ? N : BEAGLE_OP_NONE;
            for (int rep = 0; rep < 6 && rc == BEAGLE_SUCCESS; ++rep) {
                const auto t0 = std::chrono::steady_clock::now();
                rc = beagleUpdateTransitionMatrices(inst, 0, probIdx.data(), nullptr, nullptr, lengths.data(), n - 1);
                if (rc == BEAGLE_SUCCESS)
                    rc = beagleUpdatePartials(inst, reinterpret_cast<const BeagleOperation*>(ops.data()), N - 1, BEAGLE_OP_NONE);
                if (rc == BEAGLE_SUCCESS && rescale) {
                    rc = beagleResetScaleFactors(inst, cum);
                    if (rc == BEAGLE_SUCCESS) rc = beagleAccumulateScaleFactors(inst, scaleIdx.data(), N - 1, cum);
                }
                if (rc == BEAGLE_SUCCESS) {
                    rc = beagleCalculateRootLogLikelihoods(inst, &root, &zero, &zero, &cum, 1, &logL);
                    if (rc == BEAGLE_ERROR_FLOATING_POINT) rc = BEAGLE_SUCCESS;      // an underflowing synthetic tree still times
                }
                const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
                if (rep >= 2 && (best == 0.0 || ms < best)) best = ms;              // two warm-up rounds
            }
            br.returnCode = rc;
            br.benchmarkResult = best;
            beagleFinalizeInstance(inst);
        }
        results.push_back(br);
    }
    std::stable_sort(results.begin(), results.end(), [](const BeagleBenchmarkedResource& a, const BeagleBenchmarkedResource& b) {
        const bool oa = a.returnCode == BEAGLE_SUCCESS, ob = b.returnCode == BEAGLE_SUCCESS;
        return oa != ob ? oa : (oa && a.benchmarkResult < b.benchmarkResult);
    });
    for (BeagleBenchmarkedResource& r : results)
        r.performanceRatio = (results[0].benchmarkResult > 0.0 && r.returnCode == BEAGLE_SUCCESS)
                                 ? r.benchmarkResult / results[0].benchmarkResult : 0.0;
    list.list = results.data();
    list.length = (int)results.size();
    return list.length > 0 ? &list : nullptr;
}

// devices of the pattern-sharded resource for instances created from now on (default: every GPU; a device may repeat)
int b200SetShardDevices(const int* devices, int count) {
    beagleGetResourceList();
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
    if (count < 1 || count > kMaxGroup || gShardResource < 0) return BEAGLE_ERROR_OUT_OF_RANGE;
    for (int k = 0; k < count; ++k) if (devices[k] < 0 || devices[k] >= n) return BEAGLE_ERROR_OUT_OF_RANGE;
    std::lock_guard<std::mutex> lock(gMutex);
    gShardDevices.assign(devices, devices + count);
    return BEAGLE_SUCCESS;
}

// how many evaluations of this instance ran as ONE fused launch (incr.cu); -1 for an unknown instance
long b200GetFusedLaunches(int instance) {
    Instance* in = getInstance(instance);
    return in == nullptr ? -1 : in->fusedLaunches;
}

void* b200HostAlloc(long bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, (size_t)bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}

void b200HostFree(void* p) { if (p) cudaFreeHost(p); }

int b200RootLogLikelihoodsByPartitionDevice(int instance, const int* bufferIndices, const int* categoryWeightsIndices,
                                            const int* stateFrequenciesIndices, const int* cumulativeScaleIndices,
                                            const int* partitionIndices, int partitionCount, void** outDevicePointer,
                                            void** outStream) {
    GET_INSTANCE(in, instance);
    int rc = rootByPartitionLaunch(in, bufferIndices, categoryWeightsIndices, stateFrequenciesIndices,
                                   cumulativeScaleIndices, partitionIndices, partitionCount);
    if (rc != BEAGLE_SUCCESS) return rc;
    if (outDevicePointer) *outDevicePointer = in->dOut;
    if (outStream) *outStream = in->stream;
    return BEAGLE_SUCCESS;
}

int b200RootLogLikelihoodDevice(int instance, int bufferIndex, int categoryWeightsIndex, int stateFrequenciesIndex,
                                int cumulativeScaleIndex, void** outDevicePointer, void** outStream) {
    GET_INSTANCE(in, instance);
    int rc = rootLaunch(in, bufferIndex, categoryWeightsIndex, stateFrequenciesIndex, cumulativeScaleIndex, 0, in->P,
                        in->dOut, true);
    if (rc != BEAGLE_SUCCESS) return rc;
    if (outDevicePointer) *outDevicePointer = in->dOut;
    if (outStream) *outStream = in->stream;
    return BEAGLE_SUCCESS;
}

}  // extern "C"
