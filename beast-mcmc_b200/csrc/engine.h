// engine.h -- internal types of the tree-likelihood engine (not part of the ABI).
//
// One Instance owns every device allocation between beagleCreateInstance and
// beagleFinalizeInstance.  Device layout (DESIGN.md "Data layout in HBM"):
//   partials buffer   [C][Ppad][Sp] f64, or f32 on a PRECISION_SINGLE instance   (Ppad = P rounded up to 32 patterns,
//                     Sp = padded states)
//   compact tip       [Ppad] u8 + [Ppad] i32, value S = gap/unknown
//   transition matrix [C][Sp(child j)][Sp(parent i)] f64  -- stored TRANSPOSED so that a compact-tip
//                     child reads one contiguous column and lanes indexed by parent state are coalesced
//   scale buffer      [Ppad] f64 (raw factors, or logs under SCALERS_LOG; cumulative buffers: logs)
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <mutex>
#include <vector>

namespace b200 {

// op record of the generic (S > 4) walk; those instances are always double
struct alignas(16) DevOp {
    double* dest;
    const double* c1;      // child-1 partials, or nullptr when the child is a compact tip
    const double* c2;
    const void* s1;        // child-1 compact states (u8 for the 4-state path, i32 otherwise)
    const void* s2;
    const double* m1;      // transposed matrices of the two branches
    const double* m2;
    double* scaleWrite;    // nullptr = BEAGLE_OP_NONE
    const double* scaleRead;
    double* cumScale;
    int pBegin, pEnd;      // pattern range the op applies to (a partition, or [0,P))
    int srcSlot1, srcSlot2;  // operand-stack slots (4-state stack walk); -1 = read from global
    int dstSlot;             // operand-stack slot the result is parked in; -1 = none
    int pad_;
};

// Compact operation record of the 4-state walk: 64 bytes = four warp-uniform 128-bit loads, all
// addressing by index so that no pointer has to be chased on the per-op critical path.
//   dest/c1/c2 : partials slot (>= 0) in the contiguous slab, or -(tipIndex+1) for a compact tip; a virtual cherry
//                child (pad_ bit 2 / 3) is its buffer index, i.e. its row of the recipe table, and its two tips are entry
//                k of a parallel int4 array (child 1: x, y; child 2: z, w) that only k_walk4pv reads
//   m1/m2      : transition-matrix buffer index;  sw/sr/cum : scale buffer index or -1
//   slots      : byte0 srcSlot1, byte1 srcSlot2, byte2 dstSlot of the shared-memory operand stack (0xFF = none)
//   pad_       : bit 0 = pre-order op, bit 1 = child 1 is the previous op's result (taken from registers),
//                bit 2 / 3 = child 1 / 2 is a virtual cherry (read by k_walk4pv only, walk4e.cu)
//   pfA/pfB    : operands of the NEXT op of the walk that are already final in memory, prefetched into L1 while this
//                op computes: 0 = none, ((slot + 1) << 1) = partials slot, (tip << 1) | 1 = compact tip states
//   pfM1/pfM2  : the next op's matrix buffers (-1 = none)
struct alignas(16) Op4 {
    int dest, c1, c2, m1;
    int m2, sw, sr, cum;
    int pBegin, pEnd;
    unsigned int slots;
    int pad_;
    int pfA, pfB, pfM1, pfM2;
};

// a virtual cherry: a partials buffer whose value is colA[state of tip1] ⊙ colB[state of tip2] (api.cu, walk4e.cu)
struct CherryRef { int buf, tip1, tip2; };

// one edge of a calculateEdgeDerivatives call
// T = the partials' storage type (float on a PRECISION_SINGLE instance); the host fills EdgeRefT<void>, the same layout
template <typename T> struct EdgeRefT { const T* post; const int* states; const T* pre; const double* D; double len; };
using EdgeRef = EdgeRefT<double>;

// a remembered execution plan: the caller's list (key) and its device-resident op records + subtree table
struct HostOp { int dest, sw, sr, c1, m1, c2, m2, part, cum; int kind = 0; };   // kind 1 = pre-order op
// in-list cumulative scaling of an updatePartials call: cum[p] += sum over `indices` of log factor[p] on [pBegin, pEnd)
struct CumGroup { int cum, pBegin, pEnd; std::vector<int> indices; };
struct CachedPlan {
    std::vector<HostOp> key;
    std::vector<CumGroup> cumGroups;
    int n = -1;
    bool byPartition = false, fourPath = false, preOrder = false;
    unsigned long epoch = 0;
    // [op records | subtree table | snapshot items of the virtual cherries | tips of the virtual children per op]
    void* dBlock = nullptr;
    size_t capacity = 0, subsOffset = 0, snapOffset = 0, tipsOffset = 0;
    // virtual cherries: the ones the list produces (not run; their recipes are snapshot first), and the children read from
    // outside the list -- as a virtual cherry (tip1 >= 0, must still be that cherry on a hit) or as stored partials
    std::vector<CherryRef> cherries, external;
    bool readsVirtual = false;                // some op record names a virtual child: needs the eigen form
    std::vector<int> phaseStart, phaseDepth, phaseSlots;      // phaseSlots: sibling-stack depth per phase
    int maxWindow = 0;
    long lastUse = 0;
    long hits = 0;
    cudaGraphExec_t graphExec = nullptr;      // the plan's phase launches as one graph launch (plans with >= 2 launches)
    bool graphFailed = false;                 // capture or instantiation failed once: plain launches from then on
    int graphEigen = -2;                      // eigen slot / generation the captured launches carry by value (-1: matrix form)
    unsigned graphEigenGen = 0;
    int graphInvalidations = 0;
    // kept for in-place updates: when only the CONTENT of the eigen system moved (a substitution-model move), the captured
    // eigen-form walk launches get new V / V^-1 through cudaGraphExecKernelNodeSetParams instead of a re-capture
    cudaGraph_t graph = nullptr;
    std::vector<cudaGraphNode_t> graphKernelNodes;
    bool graphAllEigen = false;
    void dropGraph() {
        if (graphExec) cudaGraphExecDestroy(graphExec);
        if (graph) cudaGraphDestroy(graph);
        graphExec = nullptr; graph = nullptr; graphKernelNodes.clear(); graphAllEigen = false;
    }
};

enum TimingClass { T_PARTIALS = 0, T_MATRICES = 1, T_ROOT = 2, T_CLASSES = 3 };

// ---- deferred small evaluations (incr.cu): a short updateTransitionMatrices -> updatePartials -> root sequence as ONE
// launch, all of its arguments by value in the kernel parameters
constexpr int kIncMaxOps = 64, kIncMaxMats = 8;
struct IncOp { int dest, c1, c2, m1, m2, sw, sr, flags; };      // m < 0: pending branch -(q+1); flags bit 0: c1 = previous result
struct IncMat { int prob, rateSet; double len; };
struct IncArgs {
    void* partials; size_t stride; const uint8_t* states; double* mats; double* evecs; double* scale;
    size_t matStride;
    int S, C, Ppad, P, logScalers, nOps, nMats, pad_;
    double V[16], Vi[16], eval[4];
    double weights[8], freqs[4], rate[kIncMaxMats][8];       // by value (host mirrors): no dependent load before the first flop
    const double* cum; const double* patternWeights;
    double* site; double* blockSums; unsigned int* counter; double* out;
    volatile double* hostOut; volatile unsigned long long* hostFlag; unsigned long long seq;
    IncMat mat[kIncMaxMats];
    IncOp op[kIncMaxOps];
};

// ---- cross-GPU sum of the per-shard log-likelihoods, fused into k_root (no NCCL launch, no host in the loop) -------------
// Every member of a reduce group owns [2 banks][size] slots in ITS device memory; all members map all members' slots
// (peer access inside a process, CUDA IPC across processes).  The finishing block of k_root stores {local sum, sequence
// number} into slot [bank][rank] of EVERY member over NVLink (value, system fence, then the sequence number), then spins
// on its own device's slots until all `size` entries carry this evaluation's sequence number and adds them in rank
// order: every member ends up with the same, deterministic joint value.  Two banks suffice: a member can only reach
// evaluation k+2 after it has seen every peer's k+1, which each peer wrote after it finished reading bank k.
constexpr int kMaxGroup = 16;
struct ExchangeSlot { double value; unsigned long long seq; };
struct Exchange {
    int rank = 0, size = 1;
    unsigned long long seq = 0;              // sequence number of THIS evaluation (host-incremented per root launch)
    long long timeoutCycles = 0;             // spin budget (SM clocks) before giving up with NaN
    ExchangeSlot* peers[kMaxGroup] = {};     // member q's slot array as mapped on this device (peers[rank] = own)
};

// slots per warp of the sibling stack (built into the CP = 4 staged walk at its default launch bound of 3 blocks only,
// walk4e.cu::stackBuilt): at R = 4 one slot is 4 KB per warp, and three of them keep the 3 blocks per SM the registers allow
// inside the 228 KB of shared memory; in the cfg-2 and Makona-like plans three slots hold every sibling a walk reads back
constexpr int kStackSlots = 3;

struct Instance {
    int id = -1, device = 0, resource = 0;
    int tipCount = 0, nPartials = 0, nCompact = 0, S = 0, P = 0, nEigen = 0, nMatrices = 0, C = 0, nScale = 0;
    int Sp = 0, Ppad = 0, nBuffers = 0, nSets = 1;
    long flags = 0;
    bool logScalers = false, complexEigen = false;
    cudaStream_t stream = nullptr;
    int smCount = 132;                        // H100 SXM; replaced by the device's count at instance creation
    size_t maxSmemOptin = 0;

    // PRECISION_SINGLE (S <= 4, C <= 8): partials are stored as fp32 and every value is rounded to fp32 before it is read;
    // arithmetic, matrices, scale buffers and everything at the API stay fp64 (DESIGN.md section 4.1)
    bool single = false;
    size_t partialsElems = 0;                 // C*Ppad*Sp = stride of one partials slot, in elements
    size_t elemBytes() const { return single ? sizeof(float) : sizeof(double); }
    char* partialsBase = nullptr;             // ONE contiguous slab of nSlots partials buffers
    int nSlots = 0, nextSlot = 0;
    std::vector<int> slotOf;                  // buffer index -> slot (assigned on first use), -1 = none
    std::vector<char*> partials;              // = partialsBase + slot*stride*elemBytes(), nullptr while unassigned
    uint8_t* states8Base = nullptr;           // [tipCount][Ppad] compact states (4-state path)
    int* states32Base = nullptr;              // [tipCount][Ppad] compact states (generic path)
    std::vector<uint8_t*> states8;            // non-null while buffer idx is a compact tip
    std::vector<int*> states32;
    int matCP = 0;                            // 4-state matrix layout [j][CP][i] (CP = padded categories), 0 = [c][j][i]
    size_t matStride = 0;                     // elements per transition-matrix buffer

    double* dEigen = nullptr;                 // [nEigen][2*S*S + 2*S]
    double* dMat = nullptr;                   // [nMatrices][C][Sp][Sp] transposed
    double* dEvec = nullptr;                  // 4-state path: [nMatrices][CP][4] spectra exp(lambda_k r_c t) (walk4e.cu)
    // provenance of every matrix buffer: the eigen slot and its generation at updateTransitionMatrices time (-1 = set
    // directly / convolved); the eigen-form walk serves a list only while all its matrices stem from the CURRENT content
    // of one real eigen slot
    std::vector<int> matEigen;
    std::vector<unsigned> matEigenGen, eigenGen;
    std::vector<char> eigenReal;
    std::vector<char> eigenKind;              // any S: 0 = slot never set, 1 = real, 2 = holds complex pairs
    std::vector<double> hEigen;               // [nEigen][32]: V | V^-1 padded to 4 x 4 (host copy, by value into the launch)
    int eigenWalk = 1;                        // B200_EIGEN_WALK: 0 = always the matrix-form kernel
    int tipMode = 2;                          // B200_TIP_MODE: compact tips by contraction (0), P column from global (1), shared-memory column table (2)
    int thinTipMode = 3;                     // the same choice for thin (R = 1) phases (B200_THIN_TIP_MODE)
    // virtual cherries (B200_VIRTUAL_CHERRIES, 4-state CP <= 8): per buffer the tips of the cherry it holds (-1 = real
    // partials) and whether its partials have been written too; recipe rows [buffer][2][16 * CP]
    int virtualCherries = 1;
    std::vector<int> cherryTip1, cherryTip2;
    std::vector<char> cherryStored;
    double* dRecipe = nullptr;
    double* dRates = nullptr;                 // [nSets][C]
    std::vector<double> hRates, hWeights, hFreqs;   // host mirrors ([nSets][C], [nSets][C], [nSets][4]; 4-state instances use them)
    double* dWeights = nullptr;               // [nSets][C]
    double* dFreqs = nullptr;                 // [nSets][Sp]
    double* dScale = nullptr;                 // [nScale][Ppad]
    std::vector<char> scaleIsLog;             // per scale buffer: holds logarithms (cumulative buffers always do)
    double* dPatternWeights = nullptr;        // [Ppad], zero padded
    int* dPatternPartitions = nullptr;        // [Ppad]
    double* dSite = nullptr;                  // [Ppad]
    double* dBlockSums = nullptr;
    double* dOut = nullptr;                   // [maxPartitions + 1]
    unsigned int* dCounter = nullptr;
    int lookaheadPre = 1;                     // look-ahead prefetch in pre-order walks too (B200_LOOKAHEAD_PRE)
    int prePhases = 1;                        // pre-order lists as phased subtree walks (0: one launch per depth level)
    int useGraphs = 1;                        // B200_GRAPHS
    int lookahead = 1;                        // L1 prefetch of the next op's operands (B200_LOOKAHEAD)
    int forward = 1;                          // register forwarding between consecutive ops of a walk (B200_FORWARD)
    // slots per warp of the staged eigen walk's sibling stack (api.cu::assignStackSlots); B200_WALK_STACK_SLOTS=0 turns
    // it off, the reference route of the bit-equality tests
    int stackSlots = kStackSlots;
    bool debugLog = false;                    // B200_BEAGLE_DEBUG: per-launch diagnostics on stderr
    double* dScratch = nullptr;               // grow-only workspace of the derivative calls
    size_t scratchDoubles = 0;
    int partitionCount = 1;
    std::vector<int> partBegin, partEnd;      // contiguous pattern ranges per partition
    std::vector<int> hostPartitions;

    // pinned staging ring for the small per-call arrays (ops, indices, branch lengths)
    char* hStage = nullptr;
    char* dStage = nullptr;
    char* hStageDev = nullptr;                // hStage as the device addresses it (mapped pinned memory)
    size_t stageSize = 0, stagePos = 0;
    double* hOut = nullptr;                   // pinned result landing zone

    // deferred small evaluations (incr.cu): what updateTransitionMatrices / updatePartials have accepted but not launched yet
    int fuseSmall = 1;                        // B200_FUSE
    struct PendingMat { int prob, eigen, rateSet; double len; };
    std::vector<PendingMat> pendingMats;
    std::vector<HostOp> pendingOps;
    int pendingCum = -1;
    double* hMapped = nullptr;                // mapped pinned: [0] = value, [1] = sequence flag (as u64)
    double* dMapped = nullptr;                // its device alias
    double* dIncSums = nullptr;               // per-block partial sums of k_incremental
    unsigned int* dIncCounter = nullptr;
    unsigned long long incSeq = 0;
    long fusedLaunches = 0;

    void* shard = nullptr;                    // non-null: this id is a pattern-sharded instance over several GPUs (multi.cu)
    // reduce group (b200Exchange*): set up once, used by every single-root launch from then on
    Exchange exchange;
    ExchangeSlot* dSlots = nullptr;           // own slots [2][size]
    std::vector<void*> ipcOpened;             // peers' slot arrays opened through CUDA IPC (closed at finalize)
    bool exchangeOn = false;

    // kernel timing (bench.py roofline): events around every launch of a class
    bool timing = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> timed[T_CLASSES];
    double timedMs[T_CLASSES] = {0, 0, 0};
    long timedLaunches[T_CLASSES] = {0, 0, 0};

    // tuning knobs (environment overridable, see api.cu)
    size_t walkSmemConfigured = 0, genericSmemConfigured = 0, mmaSmemConfigured[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int walkBlock = 128;
    int walkVariant = 0;
    std::vector<CachedPlan> planCache;
    int planCacheSize = 4;
    long planClock = 0;
    unsigned long bufferEpoch = 0;     // bumped whenever a buffer changes kind (tip <-> partials) or partitions change
    int reorder = 1;
    int thinR1 = 1;              // thin (latency-bound) phases of the 4-state walk use one pattern group per thread
    int stackTail = 0;           // operand stack for latency-bound (thin) phases of the 4-state walk (experiment, off)
    int stackDepthMax = 12;
    int walkMinBlocks = 4;       // __launch_bounds__(128, n) variant of the 4-state walk (4, 5 or 6)
    bool walkMinBlocksSet = false;   // B200_WALK_MINB given explicitly
    int mmaWarps = 4;            // codon-size tensor walk: 4 warps single-buffered (default) or 8 warps double-buffered
    int tensorR = 2;             // 8-pattern tiles per warp in the 4-state tensor walk (2 or 4)
    int genericMma = 1;          // S > 4: 1 = fp64 tensor-core block walk, 0 = FMA block walk
    int walkR = 4;               // patterns per thread in the 4-state walk (1, 2 or 4)
    int phaseTmin = 4, phaseOversub = 0, phaseSmall = 24;   // phaseSmall: a remainder this short runs as one launch
    int phaseT = 0;              // max ops per subtree walk (0 = automatic)
};

// ---- multi-GPU layer (multi.cu) --------------------------------------------------------------------
struct Sharded;
Instance* instanceById(int id);               // api.cu: nullptr when the id is free
void exchangeRelease(Instance* in);
int shardedCreate(Instance* parent, int g, const int* devices, int tipCount, int partialsBufferCount, int compactBufferCount,
                  int stateCount, int patternCount, int eigenBufferCount, int matrixBufferCount, int categoryCount,
                  int scaleBufferCount, long preferenceFlags, long requirementFlags, void* details /* BeagleInstanceDetails* */);
void shardedDestroy(Instance* parent);

// ---- kernel launchers (kernels.cu) -----------------------------------------------------------
cudaError_t launchTransitionMatrices(Instance* in, const int* dProbIdx, const int* dEigenIdx,
                                     const int* dRateSet, const double* dLengths, int count);
// dSubs[k] = (first op, one-past-last op, first pattern, one-past-last pattern) of subtree walk k
cudaError_t launchWalk4(Instance* in, const Op4* dOps, const int4* dSubs, int nSubs, int stackDepth, int maxWindow, bool preOrder);
// walk4e.cu: eigen-form 4-state walk; eigen = [V (16) | V^-1 (16)]; aligned = every op covers [0, Ppad)
// new V | V^-1 (32 doubles) for the captured eigen-form walk launches of a graph; any failure = the caller re-captures
cudaError_t updateWalk4EGraph(cudaGraphExec_t exec, const std::vector<cudaGraphNode_t>& kernelNodes, const double* eigen);
// dVirtTips non-null: the records name virtual cherries whose tips are dVirtTips[op] (an error unless every phase runs on
// k_walk4p, see walk4pServes); stackSlots: slots per warp of the sibling stack the records use (k_walk4p only, 0 = none)
cudaError_t launchWalk4E(Instance* in, const Op4* dOps, const int4* dSubs, int nSubs, int maxWindow, bool aligned,
                         const double* eigen, const int4* dVirtTips, int stackSlots);
// whether an aligned eigen-form phase of nSubs subtree walks runs on k_walk4p (the kernel that reads virtual cherries)
bool walk4pServes(const Instance* in, int nSubs, int maxWindow);
// whether the staged-walk kernels this instance launches carry the sibling stack (otherwise they ignore the slot bytes)
bool walkStackBuilt(const Instance* in);
// recipe rows of the virtual cherries a list produces: items (buffer, m1, m2, -)
cudaError_t launchCherrySnapshot(Instance* in, const int4* dItems, int count);
// stored partials of virtual cherries: items (slot, buffer, tip 1, tip 2)
cudaError_t launchCherryStore(Instance* in, const int4* dItems, int count);
cudaError_t launchWalkGeneric(Instance* in, const DevOp* dOps, const int4* dSubs, int nSubs, int maxWindow, bool preOrder);
// `partial`: edgeDerivativeWorkspace() doubles when that is non-zero (tensor-pipe form), else nullptr
size_t edgeDerivativeWorkspace(const Instance* in, int count);
cudaError_t launchEdgeDerivatives(Instance* in, const EdgeRefT<void>* dEdges, int count, const double* weights, double* outPerPattern,
                                  double* outSum, double* outSumSq, double* partial);
// patterns.cu: unique site patterns in first-occurrence order (0 or a negative BEAGLE error code)
int compressSitePatterns(int device, int taxa, int sites, const int* hStates, int* hPatternOfSite, int* hPatterns,
                         double* hWeights, int* hPatternCount);
int crossProductBlocks(const Instance* in, int count);
cudaError_t launchCrossProducts(Instance* in, const EdgeRefT<void>* dEdges, int count, const double* rates,
                                const double* weights, double* scratch);
// exchange: non-null = add the other members' sums inside the kernel (dOutSlot[0] = joint value, dOutSlot[1] = local)
cudaError_t launchRoot(Instance* in, const void* root, const double* weights, const double* freqs,
                       const double* cumScale, int pBegin, int pEnd, double* dOutSlot, const Exchange* exchange = nullptr);
cudaError_t launchIncremental(Instance* in, const IncArgs& args);
cudaError_t launchCombineMatrices(Instance* in, const int* dFirst, const int* dSecond, const int* dResult, int count, bool multiply);
cudaError_t launchExchangeSum(Instance* in, const double* dVals, int n, double* dOutJoint, const Exchange* exchange);
cudaError_t launchScaleAccumulate(Instance* in, const int* dIdx, int count, double* cum, double sign,
                                  int pBegin, int pEnd);
cudaError_t launchRescalePartialsForGet(Instance* in, double* tmp, const double* cum);

// ---- joint ancestral-state sampling (ancestral.cu) ----------------------------------------------------------------------
struct AncestralArgs {
    const int4* rows;             // [row] = (partials slot, or -(tip + 1) for a compact tip; parent row; matrix buffer; 0)
    int count, P, Ppad, S, Sp, C, CP;
    int pOffset;                  // global index of pattern 0 (a shard's first pattern): the Philox counter carries it
    const void* partials;         // slab base (float on a PRECISION_SINGLE instance)
    size_t stride;                // elements per slot
    const uint8_t* states8;       // [tip][Ppad] (4-state matrix layout)
    const int* states32;          // [tip][Ppad] (generic layout)
    const double* mats;
    size_t matStride;
    const double* weights;        // [C] of the chosen set
    const double* freqs;          // [Sp] of the chosen set
    unsigned long long seed, drawIndex;
    int* outStates;               // [count][P]
    int* outCategories;           // [P]
};
cudaError_t launchAncestral(Instance* in, const AncestralArgs& args);
// api.cu: b200SampleAncestralStates on one single-device instance; patternOffset = global index of its first pattern
int sampleAncestralStates(int instance, const int* nodeBuffers, const int* parentRows, const int* matrixIndices, int count,
                          int rootBuffer, int categoryWeightsIndex, int stateFrequenciesIndex, unsigned long long seed,
                          unsigned long long drawIndex, int patternOffset, int* outStates, int* outCategories);

// ---- Markov-jump counts and rewards conditioned on the sampled states (ancestral.cu, DESIGN.md §7.2) ---------------------
constexpr int kMaxJumpRegisters = 8;
struct MarkovJumpArgs {
    int G;                        // registers
    const double* eigen;          // the eigen slot: V [S][S] | V^-1 [S][S] | eigenvalues (real parts first)
    const double* rates;          // [C] of the chosen rate set
    const double* lengths;        // [count] edge lengths (row 0 not read)
    const double* registers;      // M [G][S][S]
    double* W;                    // [G][S][S] scratch: V^-1 M_g V
    double* cond;                 // [G][count][C][S][S] conditional matrices N (row 0 unused)
    double* perRow;               // [G][count][P] n of every (row, pattern) for the branch totals, or nullptr
    double* branch;               // [G][count] or nullptr
    double* pattern;              // [G][P] or nullptr
    const double* patternWeights; // [Ppad]
};
// false when one (row, category) block of the conditional-matrix kernel does not fit in shared memory (S above 154 on an H100)
bool markovJumpsFit(const Instance* in);
cudaError_t launchMarkovJumps(Instance* in, const AncestralArgs& a, const MarkovJumpArgs& m);
// api.cu: b200SampleMarkovJumps on one single-device instance; patternOffset as for sampleAncestralStates
int sampleMarkovJumps(int instance, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                      const double* edgeLengths, int count, int rootBuffer, int categoryWeightsIndex, int stateFrequenciesIndex,
                      int eigenIndex, int categoryRatesIndex, const double* registerMatrices, int registerCount,
                      unsigned long long seed, unsigned long long drawIndex, int patternOffset, int* outStates,
                      int* outCategories, double* outBranchCounts, double* outPatternCounts);

}  // namespace b200
