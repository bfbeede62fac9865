/*
 * libhmsbeagle_b200.h -- the drop-in boundary of the H100 tree-likelihood engine.
 *
 * BEAST (beast-dev/beast-mcmc) reaches its likelihood arithmetic through
 *     beagle.Beagle (interface, lib/beagle.jar)  ->  beagle.BeagleJNIWrapper (47 natives)
 *       ->  libhmsbeagle-jni.so  ->  libhmsbeagle.so (C API "beagle.h" of beagle-dev/beagle-lib v3/v4)
 * Neither shared library nor beagle.h is vendored in the reference (SURVEY.md 0.2).  This header
 * declares the C functions our libhmsbeagle.so exports under the upstream names so that (a) our own
 * JNI shim (csrc/jni_shim.cpp) and (b) any program written against upstream beagle.h binds to it.
 * Prototypes are restated from the parameter lists the jar's natives carry
 * (tests/golden/beagle_jar_abi.json, generated from lib/beagle.jar) and from the reference call
 * sites cited per function.  "BDLD" = src/dr/evomodel/treedatalikelihood/BeagleDataLikelihoodDelegate.java,
 * "HSMD" = .../HomogenousSubstitutionModelDelegate.java, "MPDLD" = .../MultiPartitionDataLikelihoodDelegate.java,
 * "BTL" = src/dr/evomodel/treelikelihood/BeagleTreeLikelihood.java.
 *
 * Conventions (SURVEY.md 8b): all arrays are caller-owned and only valid during the call; buffers
 * are addressed by small integers chosen by the caller, -1 (BEAGLE_OP_NONE) = "no buffer"; every
 * function returns a BeagleReturnCodes value (>= 0 instance id for beagleCreateInstance); no C++
 * exception crosses this boundary.  Layouts are row-major: partials [category][pattern][state],
 * transition matrices [category][parentState][childState], eigenvectors [S][S].
 */
#ifndef LIBHMSBEAGLE_B200_H
#define LIBHMSBEAGLE_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define BEAGLE_DLLEXPORT __attribute__((visibility("default")))
#else
#define BEAGLE_DLLEXPORT
#endif

/* beagle.BeagleErrorCode (decoded from the jar) */
enum BeagleReturnCodes {
    BEAGLE_SUCCESS = 0,
    BEAGLE_ERROR_GENERAL = -1,
    BEAGLE_ERROR_OUT_OF_MEMORY = -2,
    BEAGLE_ERROR_UNIDENTIFIED_EXCEPTION = -3,
    BEAGLE_ERROR_UNINITIALIZED_INSTANCE = -4,
    BEAGLE_ERROR_OUT_OF_RANGE = -5,
    BEAGLE_ERROR_NO_RESOURCE = -6,
    BEAGLE_ERROR_NO_IMPLEMENTATION = -7,
    BEAGLE_ERROR_FLOATING_POINT = -8
};

/* beagle.BeagleFlag masks (decoded from the jar; note the shipped collision at bit 30) */
/* plain macros: the masks exceed the range of a C enum (bit 32, 33) */
#define BEAGLE_FLAG_PRECISION_SINGLE (1L << 0)
#define BEAGLE_FLAG_PRECISION_DOUBLE (1L << 1)
#define BEAGLE_FLAG_COMPUTATION_SYNCH (1L << 2)
#define BEAGLE_FLAG_COMPUTATION_ASYNCH (1L << 3)
#define BEAGLE_FLAG_EIGEN_REAL (1L << 4)
#define BEAGLE_FLAG_EIGEN_COMPLEX (1L << 5)
#define BEAGLE_FLAG_SCALING_MANUAL (1L << 6)
#define BEAGLE_FLAG_SCALING_AUTO (1L << 7)
#define BEAGLE_FLAG_SCALING_ALWAYS (1L << 8)
#define BEAGLE_FLAG_SCALERS_RAW (1L << 9)
#define BEAGLE_FLAG_SCALERS_LOG (1L << 10)
#define BEAGLE_FLAG_VECTOR_SSE (1L << 11)
#define BEAGLE_FLAG_VECTOR_NONE (1L << 12)
#define BEAGLE_FLAG_THREADING_OPENMP (1L << 13)
#define BEAGLE_FLAG_THREADING_NONE (1L << 14)
#define BEAGLE_FLAG_PROCESSOR_CPU (1L << 15)
#define BEAGLE_FLAG_PROCESSOR_GPU (1L << 16)
#define BEAGLE_FLAG_PROCESSOR_FPGA (1L << 17)
#define BEAGLE_FLAG_PROCESSOR_CELL (1L << 18)
#define BEAGLE_FLAG_SCALING_DYNAMIC (1L << 19)
#define BEAGLE_FLAG_FRAMEWORK_CUDA (1L << 22)
#define BEAGLE_FLAG_FRAMEWORK_OPENCL (1L << 23)
#define BEAGLE_FLAG_FRAMEWORK_CPU (1L << 27)
#define BEAGLE_FLAG_PARALLELOPS_STREAMS (1L << 28)
#define BEAGLE_FLAG_PARALLELOPS_GRID (1L << 29)
#define BEAGLE_FLAG_THREADING_CPP (1L << 30)
#define BEAGLE_FLAG_PREORDER_TRANSPOSE_MANUAL (1L << 30)
#define BEAGLE_FLAG_PREORDER_TRANSPOSE_AUTO (1L << 31)
#define BEAGLE_FLAG_PREORDER_TRANSPOSE_LOW_MEMORY (1L << 32)
#define BEAGLE_FLAG_VECTOR_TENSOR (1L << 33)
#define BEAGLE_BENCHFLAG_SCALING_NONE (1L << 0)
#define BEAGLE_BENCHFLAG_SCALING_ALWAYS (1L << 1)
#define BEAGLE_BENCHFLAG_SCALING_DYNAMIC (1L << 2)

enum BeagleOpCodes { BEAGLE_OP_COUNT = 7, BEAGLE_PARTITION_OP_COUNT = 9, BEAGLE_OP_NONE = -1 };

/* beagle.InstanceDetails (setResourceNumber/setFlags/setResourceName/setImplementationName) */
typedef struct {
    int resourceNumber;
    char* resourceName;
    char* implName;
    char* implDescription;
    long flags;
} BeagleInstanceDetails;

/* beagle.ResourceDetails; BEAST prints description split on '|' (BDLD:463-470) */
typedef struct {
    char* name;
    char* description;
    long supportFlags;
    long requiredFlags;
} BeagleResource;

typedef struct {
    BeagleResource* list;
    int length;
} BeagleResourceList;

/* beagle.BenchmarkedResourceDetails (BDLD:413-434) */
typedef struct {
    int number;
    char* name;
    char* description;
    long supportFlags;
    long requiredFlags;
    int returnCode;
    char* implName;
    long benchedFlags;
    double benchmarkResult;
    double performanceRatio;
} BeagleBenchmarkedResource;

typedef struct {
    BeagleBenchmarkedResource* list;
    int length;
} BeagleBenchmarkedResourceList;

/* beagle.Beagle.OPERATION_TUPLE_SIZE = 7 ints, filled at BDLD:857-902 */
typedef struct {
    int destinationPartials;
    int destinationScaleWrite;
    int destinationScaleRead;
    int child1Partials;
    int child1TransitionMatrix;
    int child2Partials;
    int child2TransitionMatrix;
} BeagleOperation;

/* PARTITION_OPERATION_TUPLE_SIZE = 9 ints, filled at MPDLD:972-981 */
typedef struct {
    int destinationPartials;
    int destinationScaleWrite;
    int destinationScaleRead;
    int child1Partials;
    int child1TransitionMatrix;
    int child2Partials;
    int child2TransitionMatrix;
    int partition;
    int cumulativeScaleIndex;
} BeagleOperationByPartition;

/* ---- library / resources ------------------------------------------------------------------- */
/* native getVersion(): must parse as (\d+)\.(\d+)\.(\d+).* with major >= 4
 * (src/dr/app/beast/BeastMain.java:945-950, BeagleFunctionality.java:53-71). */
BEAGLE_DLLEXPORT const char* beagleGetVersion(void);
BEAGLE_DLLEXPORT const char* beagleGetCitation(void);
/* native getResourceList(): 0 = host fallback (reported, not implemented: creating on it yields
 * BEAGLE_ERROR_NO_RESOURCE), 1..N = the visible GPUs ("0 == CPU", BDLD:71-73,275-281). */
BEAGLE_DLLEXPORT BeagleResourceList* beagleGetResourceList(void);
/* native getBenchmarkedResourceList (BDLD:413-426, -beagle_auto) */
BEAGLE_DLLEXPORT BeagleBenchmarkedResourceList* beagleGetBenchmarkedResourceList(
    int tipCount, int compactBufferCount, int stateCount, int patternCount, int categoryCount,
    int* resourceList, int resourceCount, long preferenceFlags, long requirementFlags,
    int eigenModelCount, int partitionCount, int calculateDerivatives, long benchmarkFlags);

/* ---- instance life cycle --------------------------------------------------------------------- */
/* BeagleFactory.loadBeagleInstance -> native createInstance (BDLD:439-452; MPDLD:455-470; BTL:380-400) */
BEAGLE_DLLEXPORT int beagleCreateInstance(int tipCount, int partialsBufferCount, int compactBufferCount,
                                          int stateCount, int patternCount, int eigenBufferCount,
                                          int matrixBufferCount, int categoryCount, int scaleBufferCount,
                                          int* resourceList, int resourceCount, long preferenceFlags,
                                          long requirementFlags, BeagleInstanceDetails* returnInfo);
/* Beagle.finalize() (BDLD:1234-1261) */
BEAGLE_DLLEXPORT int beagleFinalizeInstance(int instance);
BEAGLE_DLLEXPORT int beagleFinalize(void);
/* Beagle.setCPUThreadCount (BDLD:482-499); accepted and ignored on a GPU instance */
BEAGLE_DLLEXPORT int beagleSetCPUThreadCount(int instance, int threadCount);

/* ---- data upload ----------------------------------------------------------------------------- */
/* Beagle.setTipStates(tip, int[P]) (BDLD:712-726); state >= stateCount means gap/unknown */
BEAGLE_DLLEXPORT int beagleSetTipStates(int instance, int tipIndex, const int* inStates);
BEAGLE_DLLEXPORT int beagleGetTipStates(int instance, int tipIndex, int* outStates);
/* Beagle.setTipPartials(tip, double[P*S]) -- replicated over categories by the engine */
BEAGLE_DLLEXPORT int beagleSetTipPartials(int instance, int tipIndex, const double* inPartials);
/* Beagle.setPartials(buffer, double[C*P*S]) (BDLD:638-702) */
BEAGLE_DLLEXPORT int beagleSetPartials(int instance, int bufferIndex, const double* inPartials);
/* Beagle.getPartials(buffer, scaleIndex, double[C*P*S]) (BDLD:1026-1030) */
BEAGLE_DLLEXPORT int beagleGetPartials(int instance, int bufferIndex, int scaleIndex, double* outPartials);
/* Beagle.setEigenDecomposition(idx, Evec, Ievc, Eval) (HSMD:228-239; SubstitutionModelDelegate.java:272-287).
 * Eval holds S reals, or 2S (real || imaginary) when the instance was created with EIGEN_COMPLEX. */
BEAGLE_DLLEXPORT int beagleSetEigenDecomposition(int instance, int eigenIndex, const double* inEigenVectors,
                                                 const double* inInverseEigenVectors,
                                                 const double* inEigenValues);
/* Beagle.setStateFrequencies(idx, double[S]) (BDLD:832-835) */
BEAGLE_DLLEXPORT int beagleSetStateFrequencies(int instance, int stateFrequenciesIndex,
                                               const double* inStateFrequencies);
/* Beagle.setCategoryWeights(idx, double[C]) (BDLD:827-829) */
BEAGLE_DLLEXPORT int beagleSetCategoryWeights(int instance, int categoryWeightsIndex,
                                              const double* inCategoryWeights);
/* Beagle.setCategoryRates(double[C]) (BDLD:819-825) / setCategoryRatesWithIndex (MPDLD:835) */
BEAGLE_DLLEXPORT int beagleSetCategoryRates(int instance, const double* inCategoryRates);
BEAGLE_DLLEXPORT int beagleSetCategoryRatesWithIndex(int instance, int categoryRatesIndex,
                                                     const double* inCategoryRates);
/* Beagle.setPatternWeights(double[P]) (BDLD:535) */
BEAGLE_DLLEXPORT int beagleSetPatternWeights(int instance, const double* inPatternWeights);
/* Beagle.setPatternPartitions(partitionCount, int[P]) (MPDLD:552-553) */
BEAGLE_DLLEXPORT int beagleSetPatternPartitions(int instance, int partitionCount, const int* inPatternPartitions);

/* ---- transition matrices --------------------------------------------------------------------- */
/* Beagle.updateTransitionMatrices(eigenIndex, probIdx[n], d1=null, d2=null, t[n], n) (HSMD:247-266):
 * P_c(t) = Evec . diag(exp(Eval . rate_c . t)) . Ievc  per branch, per rate category. */
BEAGLE_DLLEXPORT int beagleUpdateTransitionMatrices(int instance, int eigenIndex, const int* probabilityIndices,
                                                    const int* firstDerivativeIndices,
                                                    const int* secondDerivativeIndices,
                                                    const double* edgeLengths, int count);
/* MPDLD:880-887 */
BEAGLE_DLLEXPORT int beagleUpdateTransitionMatricesWithMultipleModels(
    int instance, const int* eigenIndices, const int* categoryRateIndices, const int* probabilityIndices,
    const int* firstDerivativeIndices, const int* secondDerivativeIndices, const double* edgeLengths, int count);
/* Beagle.setTransitionMatrix / getTransitionMatrix (preorder/AbstractBeagleGradientDelegate.java:96-99) */
BEAGLE_DLLEXPORT int beagleSetTransitionMatrix(int instance, int matrixIndex, const double* inMatrix,
                                               double paddedValue);
BEAGLE_DLLEXPORT int beagleGetTransitionMatrix(int instance, int matrixIndex, double* outMatrix);
/* Beagle.setDifferentialMatrix(idx, double[C*S*S]) (HomogenousSubstitutionModelDelegate.java:160-176): same storage as a
 * transition matrix; consumed by beagleCalculateEdgeDerivatives */
BEAGLE_DLLEXPORT int beagleSetDifferentialMatrix(int instance, int matrixIndex, const double* inMatrix);
/* SubstitutionModelDelegate.java:303-470 (epoch models) */
BEAGLE_DLLEXPORT int beagleConvolveTransitionMatrices(int instance, const int* firstIndices,
                                                      const int* secondIndices, const int* resultIndices,
                                                      int matrixCount);
BEAGLE_DLLEXPORT int beagleAddTransitionMatrices(int instance, const int* firstIndices, const int* secondIndices,
                                                 const int* resultIndices, int matrixCount);
BEAGLE_DLLEXPORT int beagleTransposeTransitionMatrices(int instance, const int* inputIndices,
                                                       const int* resultIndices, int matrixCount);

/* ---- partials -------------------------------------------------------------------------------- */
/* Beagle.updatePartials(int[7n], n, cumulativeScaleIndex) (BDLD:857-904; BTL:997-1003):
 * dest[c,p,i] = (sum_j M1[c,i,j] child1[c,p,j]) * (sum_j M2[c,i,j] child2[c,p,j]); compact-tip
 * children contribute M[c,i,state_p] (1 if state >= S); then per-pattern max rescale into
 * destinationScaleWrite, or division by the factors stored in destinationScaleRead. */
BEAGLE_DLLEXPORT int beagleUpdatePartials(int instance, const BeagleOperation* operations, int operationCount,
                                          int cumulativeScaleIndex);
/* MPDLD:972-997 */
BEAGLE_DLLEXPORT int beagleUpdatePartialsByPartition(int instance, const BeagleOperationByPartition* operations,
                                                     int operationCount);
BEAGLE_DLLEXPORT int beagleWaitForPartials(int instance, const int* destinationPartials,
                                           int destinationPartialsCount);
/* Beagle.updatePrePartials(int[7n], n, cumulativeScaleIndex) (preorder/AbstractBeagleGradientDelegate.java:120,206-220):
 * op = {pre[node], scaleWrite, scaleRead, pre[parent], matrix(node), post[sibling], matrix(sibling)};
 * pre[node][c,p,j] = sum_i ( pre[parent][c,p,i] * sum_k M_sib[c,i,k] post[sib][c,p,k] ) * M_node[c,i,j]. */
BEAGLE_DLLEXPORT int beagleUpdatePrePartials(int instance, const BeagleOperation* operations, int operationCount,
                                             int cumulativeScaleIndex);
BEAGLE_DLLEXPORT int beagleUpdatePrePartialsByPartition(int instance, const BeagleOperationByPartition* operations,
                                                        int operationCount);

/* ---- scale factors (BDLD:915-926; MPDLD:1016-1017; BTL:1019-1025,1548) --------------------------- */
BEAGLE_DLLEXPORT int beagleAccumulateScaleFactors(int instance, const int* scaleIndices, int count,
                                                  int cumulativeScaleIndex);
BEAGLE_DLLEXPORT int beagleAccumulateScaleFactorsByPartition(int instance, const int* scaleIndices, int count,
                                                             int cumulativeScaleIndex, int partitionIndex);
BEAGLE_DLLEXPORT int beagleRemoveScaleFactors(int instance, const int* scaleIndices, int count,
                                              int cumulativeScaleIndex);
BEAGLE_DLLEXPORT int beagleRemoveScaleFactorsByPartition(int instance, const int* scaleIndices, int count,
                                                         int cumulativeScaleIndex, int partitionIndex);
BEAGLE_DLLEXPORT int beagleResetScaleFactors(int instance, int cumulativeScaleIndex);
BEAGLE_DLLEXPORT int beagleResetScaleFactorsByPartition(int instance, int cumulativeScaleIndex, int partitionIndex);
BEAGLE_DLLEXPORT int beagleCopyScaleFactors(int instance, int destScalingIndex, int srcScalingIndex);
/* native getLogScaleFactors -> log of the stored factors */
BEAGLE_DLLEXPORT int beagleGetScaleFactors(int instance, int srcScalingIndex, double* outScaleFactors);
BEAGLE_DLLEXPORT int beagleGetLogScaleFactors(int instance, int srcScalingIndex, double* outLogScaleFactors);

/* ---- root integration ------------------------------------------------------------------------ */
/* Beagle.calculateRootLogLikelihoods({root},{wIdx},{fIdx},{cumScale},1,out[1]) (BDLD:928-937):
 * site[p] = log(sum_c w_c sum_i pi_i root[c,p,i]) + cum[p];  out = sum_p weight[p] site[p].
 * Returns BEAGLE_ERROR_FLOATING_POINT when out is NaN (the jar lets -8 through; BEAST tests
 * isNaN/isInfinite itself, BDLD:946). */
BEAGLE_DLLEXPORT int beagleCalculateRootLogLikelihoods(int instance, const int* bufferIndices,
                                                       const int* categoryWeightsIndices,
                                                       const int* stateFrequenciesIndices,
                                                       const int* cumulativeScaleIndices, int count,
                                                       double* outSumLogLikelihood);
/* MPDLD:1074-1083 */
BEAGLE_DLLEXPORT int beagleCalculateRootLogLikelihoodsByPartition(
    int instance, const int* bufferIndices, const int* categoryWeightsIndices, const int* stateFrequenciesIndices,
    const int* cumulativeScaleIndices, const int* partitionIndices, int partitionCount, int count,
    double* outSumLogLikelihoodByPartition, double* outSumLogLikelihood);
/* Beagle.calculateCrossProductDifferentials(post[], pre[], {ratesIdx}, {weightsIdx}, edgeLengths[], count, outSum,
 * outSumSquared) (discrete/SubstitutionModelCrossProductDelegate.java:158-176; consumed by
 * AbstractLogAdditiveSubstitutionModelGradient.java:239-270): outSum is S*S row-major and is ADDED to:
 *   outSum[i*S+j] += sum_e t_e sum_p weight_p (sum_c w_c r_c pre_e[c,p,i] post_e[c,p,j]) / (sum_c w_c pre_e[c,p,.].post_e[c,p,.])
 * outSumSquared must be NULL (BEAST passes null). */
BEAGLE_DLLEXPORT int beagleCalculateCrossProductDerivative(int instance, const int* postBufferIndices,
                                                           const int* preBufferIndices, const int* categoryRatesIndices,
                                                           const int* categoryWeightsIndices, const double* edgeLengths,
                                                           int count, double* outSumDerivatives,
                                                           double* outSumSquaredDerivatives);
/* Beagle.calculateEdgeDifferentials(post[], pre[], derivativeMatrix[], {weightsIdx}, count, out, outSum, outSumSquared)
 * (preorder/AbstractBeagleBranchGradientDelegate.java:83-91): per edge e and pattern p
 *   d[e,p] = (sum_c w_c sum_j pre[c,p,j] sum_k D[c,j,k] post[c,p,k]) / (sum_c w_c sum_j pre[c,p,j] post[c,p,j]);
 * outDerivatives[e*P + p] = d (may be NULL), outSum[e] = sum_p weight_p d, outSumSquared[e] = sum_p weight_p d^2
 * (each may be NULL).  D is a matrix buffer filled by beagleSetDifferentialMatrix. */
BEAGLE_DLLEXPORT int beagleCalculateEdgeDerivatives(int instance, const int* postBufferIndices, const int* preBufferIndices,
                                                    const int* derivativeMatrixIndices, const int* categoryWeightsIndices,
                                                    int count, double* outDerivatives, double* outSumDerivatives,
                                                    double* outSumSquaredDerivatives);
/* Beagle.getSiteLogLikelihoods(double[P]) (BDLD:1020-1024; BTL:1050-1056) */
BEAGLE_DLLEXPORT int beagleGetSiteLogLikelihoods(int instance, double* outLogLikelihoods);

/* ---- engine extensions (not in upstream beagle.h) -------------------------------------------- */
/* Timing hook for bench.py: device milliseconds spent in the engine's kernels of the named class
 * since the last reset, measured with CUDA events on the instance stream.
 * which: 0 = updatePartials kernels, 1 = updateTransitionMatrices, 2 = root/scale kernels. */
BEAGLE_DLLEXPORT int b200SetKernelTiming(int instance, int enable);
BEAGLE_DLLEXPORT int b200GetKernelTiming(int instance, int which, double* outMilliseconds, long* outLaunches);
/* SHA-256 prefix (16 hex digits) of the sources this binary was built from; __graft_entry__.build() and
 * beast-mcmc_b200/build.py compare it with the tree so that a prebuilt library cannot drift from its sources.  The same
 * string is the build-metadata suffix of beagleGetVersion ("4.0.1-b200+<hash>"). */
BEAGLE_DLLEXPORT const char* b200GetSourceHash(void);
/* Deferred small evaluations (csrc/incr.cu): on 4-state instances a short beagleUpdateTransitionMatrices (<= 8 branches) ->
 * beagleUpdatePartials (<= 64 operations, chain-like: every operation but at most two consumes its predecessor's result, or
 * <= 16 operations) -> beagleCalculateRootLogLikelihoods sequence -- what an MCMC move that dirties one or two root paths
 * issues (MarkovChain.java:207-393) -- is executed as ONE kernel launch at the root call, its result written
 * to mapped pinned host memory; any other entry point first launches what was deferred, so the calls keep their upstream
 * meaning.  B200_FUSE=0 (environment) switches the deferral off.  This counter reports how often it happened. */
BEAGLE_DLLEXPORT long b200GetFusedLaunches(int instance);
/* Pinned-host staging for callers that want the H2D/D2H copies to be asynchronous. */
BEAGLE_DLLEXPORT void* b200HostAlloc(long bytes);
BEAGLE_DLLEXPORT void b200HostFree(void* p);
/* Asynchronous variant of beagleCalculateRootLogLikelihoods for engine-internal multi-GPU use:
 * leaves the sum in device memory and returns its device pointer (no host sync). */
BEAGLE_DLLEXPORT int b200RootLogLikelihoodDevice(int instance, int bufferIndex, int categoryWeightsIndex,
                                                 int stateFrequenciesIndex, int cumulativeScaleIndex,
                                                 void** outDevicePointer, void** outStream);

/* ---- multi-GPU (SURVEY.md 8e) -----------------------------------------------------------------------------------
 * Mode B, one instance over several GPUs: beagleGetResourceList() ends with a resource "GPU x N (pattern-sharded)" on
 * boxes with >= 2 GPUs; an instance created on it splits its patterns into contiguous blocks (the rule of BEAST's own
 * -beagle_instances split, src/dr/evolution/alignment/Patterns.java:142-169) over the GPUs and behaves like any other
 * instance -- beagleCalculateRootLogLikelihoods returns the joint value (CompoundLikelihood.java:214-219 sums the same
 * shards on the Java side in mode A).  B200_SHARD_DEVICES="0,1,..." (environment) overrides the device list.
 *
 * Reduce groups, for callers that keep one instance per GPU themselves (mode A inside one JVM, or one process per GPU):
 * once connected, every beagleCalculateRootLogLikelihoods / b200RootLogLikelihoodDevice of a member returns the SUM over
 * all members -- the finishing block of the root kernel stores the shard's sum into every member's device memory over
 * NVLink and adds what the others stored (no NCCL call, no host arithmetic).  All members must issue the same number of
 * root evaluations.
 *   same process : b200ExchangeConnectLocal(instances, count)          (peer mappings)
 *   one process per GPU: b200ExchangeCreate(instance, rank, size, handle64) on every rank, exchange the 64-byte handles by
 *                  any means (bench.py: torch.distributed all_gather at set-up), then b200ExchangeConnect(instance,
 *                  all size*64 bytes in rank order)                    (CUDA IPC mappings) */
BEAGLE_DLLEXPORT int b200SetShardDevices(const int* devices, int count);   /* device list of the sharded resource from now on */
BEAGLE_DLLEXPORT int b200ExchangeConnectLocal(const int* instances, int count);
BEAGLE_DLLEXPORT int b200ExchangeCreate(int instance, int rank, int size, void* outIpcHandle64);
BEAGLE_DLLEXPORT int b200ExchangeConnect(int instance, const void* allIpcHandles64);

/* Asynchronous variant of beagleCalculateRootLogLikelihoodsByPartition: per-partition sums stay in device memory
 * ([0..partitionCount) at *outDevicePointer, followed by {joint, own total} for a member of a reduce group). */
BEAGLE_DLLEXPORT int b200RootLogLikelihoodsByPartitionDevice(int instance, const int* bufferIndices,
                                                             const int* categoryWeightsIndices,
                                                             const int* stateFrequenciesIndices,
                                                             const int* cumulativeScaleIndices, const int* partitionIndices,
                                                             int partitionCount, void** outDevicePointer, void** outStream);

/* The step before the path (SURVEY.md 8f rank 4): SitePatterns.addPatterns with CompressionType.UNIQUE_ONLY
 * (src/dr/evolution/alignment/SitePatterns.java:226-372) on the GPU.  inStates is [taxon][site] (the int state codes
 * SiteList.getSitePattern yields, any values); results: outSitePatternIndices[site], outPatterns [taxon][*outPatternCount]
 * (capacity taxonCount*siteCount ints), outWeights[pattern] = sum of site weights (inSiteWeights NULL = 1 per site; added
 * in site order like the Java), patterns numbered by first occurrence.  Not part of upstream beagle.h: a caller-side
 * change (SitePatterns) would be needed to use it from BEAST. */
BEAGLE_DLLEXPORT int b200CompressSitePatterns(int resourceNumber, int taxonCount, int siteCount, const int* inStates,
                                              const double* inSiteWeights, int* outSitePatternIndices, int* outPatterns,
                                              double* outWeights, int* outPatternCount);

/* Joint ancestral states on the device: per pattern p ONE draw of (rate category, state of every listed node) from the
 * exact joint posterior given the data, the post-order partials the instance holds and its transition matrices (what
 * AncestralStateBeagleTreeLikelihood draws in Java from getPartials / getTransitionMatrix; DESIGN.md section 7).
 * Rows in pre-order: row 0 is the root (parentRows[0] = -1; nodeBuffers[0] and matrixIndices[0] are not read), every other
 * row r names its node's post-order buffer nodeBuffers[r], its parent row parentRows[r] < r and the matrix buffer of the
 * branch above it matrixIndices[r].
 *   root : (c, i) with probability proportional to w_c * pi_i * Lroot_c[p][i]   (rootBuffer, categoryWeightsIndex,
 *          stateFrequenciesIndex)
 *   row r: j given the parent row's state i and the root's category c, proportional to P_c[i][j] * L_r,c[p][j]; a compact
 *          tip keeps its observed state, a gap / unknown state draws proportional to P_c[i][j]; tips given as partials and
 *          internal buffers use their partials
 * Each draw is an inverse CDF over the items in index order ((c, i) category-major at the root) with fp64 cumulative sums;
 * the uniform is (x >> 11) * 2^-53, x = the first output word of Philox4x64-10 (numpy.random.Philox) with key (seed, 0) and
 * counter (drawIndex, global pattern index, row, 0), so a draw depends on neither the launch geometry nor the sharding.
 * If no cumulative sum exceeds u * total (all weights zero: data impossible under the model) the last item of positive
 * weight is taken, else item 0.  Rescale factors cancel in every conditional: scale buffers are not inputs.
 * outStates[row * patternCount + p] (int, capacity count * patternCount), outCategories[p].  Returns
 * BEAGLE_ERROR_OUT_OF_RANGE, launching nothing, for a parent row not before its child, an index out of range or a buffer
 * that holds neither partials nor tip states. */
BEAGLE_DLLEXPORT int b200SampleAncestralStates(int instance, const int* nodeBuffers, const int* parentRows,
                                               const int* matrixIndices, int count, int rootBuffer, int categoryWeightsIndex,
                                               int stateFrequenciesIndex, unsigned long long seed,
                                               unsigned long long drawIndex, int* outStates, int* outCategories);
/* Markov-jump counts and rewards on the device, conditioned on ONE joint ancestral draw (what
 * MarkovJumpsBeagleTreeLikelihood computes in Java after each AncestralStateBeagleTreeLikelihood draw; Minin & Suchard 2008,
 * BEAST's MarkovJumpsCore; DESIGN.md section 7.2).
 * Rows, seed and drawIndex exactly as in b200SampleAncestralStates: the states and categories drawn are bit-identical to what
 * b200SampleAncestralStates returns for the same arguments (same Philox counters).
 *   registerMatrices [registerCount][S][S] row-major, the register-weighted rate matrices M_g the caller forms: counts
 *          M_ij = Q_ij * R_ij (i != j) with a zero diagonal, rewards M = diag(r).  The engine only sees M.
 *   eigen system: the real system in slot eigenIndex, Q = V diag(lambda) V^-1.
 *   time along the branch above row r >= 1: tau = r_c * edgeLengths[r], r_c the rate of the pattern's drawn category c in
 *          set categoryRatesIndex (edgeLengths[0] is not read).
 * For every row r >= 1, category c and register g:
 *   I_kl(tau) = tau * exp(lambda_l tau) * phi((lambda_k - lambda_l) tau), phi(x) = expm1(x) / x, phi(0) = 1
 *          (evaluated with the larger of lambda_k, lambda_l in the exponential: the same value, no overflow)
 *   W_g = V^-1 M_g V;  E = V (W_g o I(tau)) V^-1 (o: entrywise);  Phat = |V diag(exp(lambda tau)) V^-1| entrywise, in the
 *          formula and summation order of the transition matrices;  N[i][j] = E[i][j] / Phat[i][j], 0 where Phat[i][j] = 0
 *   n_g[r][p] = N_g,c,r[x_parent(r)][x_r] with c and x the drawn category and states (a compact tip's observed state is its
 *          x); row 0 contributes nothing.
 * outBranchCounts[g * count + r] = sum_p w_p n_g[r][p] (w the instance's pattern weights: the sum over sites; row 0 is 0),
 * outPatternCounts[g * patternCount + p] = sum_{r >= 1} n_g[r][p].  outStates [count][patternCount] and outCategories
 * [patternCount] as in b200SampleAncestralStates; any output may be NULL except both count outputs, and only the outputs
 * asked for are copied back.  No atomics: repeated calls are bit-identical, the branch totals are summed in a fixed order.
 * Every error returns before anything is launched (deferred work included) and leaves every output untouched:
 * BEAGLE_ERROR_OUT_OF_RANGE for whatever b200SampleAncestralStates rejects (its NULL-output rule aside), eigenIndex out of
 * range or never set, categoryRatesIndex out of range, edgeLengths == NULL or an edgeLengths[r] (r >= 1) negative or not
 * finite, registerMatrices == NULL, registerCount outside 1..8, both count outputs NULL; BEAGLE_ERROR_NO_IMPLEMENTATION
 * when the eigen slot holds complex pairs, or when S is so large that one (row, category) block of the conditional matrices
 * does not fit in the device's shared memory (S above 154 on an H100). */
BEAGLE_DLLEXPORT int b200SampleMarkovJumps(int instance, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                                           const double* edgeLengths, int count, int rootBuffer, int categoryWeightsIndex,
                                           int stateFrequenciesIndex, int eigenIndex, int categoryRatesIndex,
                                           const double* registerMatrices, int registerCount, unsigned long long seed,
                                           unsigned long long drawIndex, int* outStates, int* outCategories,
                                           double* outBranchCounts, double* outPatternCounts);
/* Complete substitution histories on the device by uniformization, conditioned on ONE joint ancestral draw (what BEAST's
 * Markov-jumps likelihood draws in Java with useUniformization / saveCompleteHistory; DESIGN.md section 7.3).  It needs only
 * the generator, so non-reversible models with complex eigenvalues are served.
 * Rows, seed and drawIndex exactly as in b200SampleAncestralStates: outStates and outCategories are bit-identical to what
 * it returns (same Philox counters (drawIndex, global pattern, row, 0)).
 *   rateMatrix [S][S] row-major, the generator Q (one per call, shared by all categories).  mu = max_i -Q_ii, R = I + Q/mu
 *          (R = I and no events when mu = 0).  tau = r_c * edgeLengths[r] for row r >= 1, r_c the rate of the pattern's
 *          drawn category c in set categoryRatesIndex.  N = ceil(mu tau_max + 12 sqrt(mu tau_max) + 12), tau_max the
 *          largest tau over rows >= 1 and all categories; the powers R^n, n = 0..N, are formed on the device once per call.
 *   Per (row r >= 1, pattern p) with parent state a and own state b:
 *     1. n, the number of uniformized jumps, drawn with weights pi_n (R^n)[a][b], n = 0..N, pi_0 = exp(-mu tau),
 *        pi_n = pi_{n-1} mu tau / n (the truncated distribution);
 *     2. s_k for k = 1..n-1 drawn with weights R[s_{k-1}][j] (R^{n-k})[j][b] over j, s_0 = a, s_n = b;
 *     3. U_0 = 0, U_k = 1 - (1 - U_{k-1}) v_k^{1/(n-k+1)} (computed as U_{k-1} - (1 - U_{k-1}) expm1(log(v_k)/(n-k+1)));
 *     4. a jump with s_k = s_{k-1} is virtual and dropped; every other is an event (time edgeLengths[r] U_k from the
 *        parent end, new state s_k).
 *     Each draw is the sampler's inverse CDF (sequential fp64 sums; the first item whose sum exceeds u * total, else the
 *     last of positive weight, else item 0).  When every weight of the n draw is 0 (b unreachable from a), n = 0.
 *     Uniform j of the pair is word j mod 4 of the Philox4x64-10 block at counter (drawIndex, global pattern, r, 1 + j/4),
 *     u = (x >> 11) 2^-53: j = 0 draws n, j = 1..n-1 the states, j = n..2n-1 are the v_k.
 *   registerMatrices [registerCount][S][S] as in b200SampleMarkovJumps (counts M_ij = Q_ij R_ij off the diagonal, rewards
 *          M = diag(r)).  n_g[r][p] = sum over events (i -> j) of M_g[i][j] / Q[i][j] + sum over segments k = 0..n of
 *          M_g[s_k][s_k] tau (U_{k+1} - U_k), U_{n+1} = 1.  An event adds the register's weight of its change and time is in
 *          tau units, so E[n_g | a, b] is the N_g[a][b] of b200SampleMarkovJumps.
 * outBranchCounts[g * count + r] = sum_p w_p n_g[r][p] (row 0 is 0); outPatternCounts[g * patternCount + p] =
 * sum_{r >= 1} n_g[r][p] in row order; outJumpCounts[r * patternCount + p] = the number of events (row 0 is 0).
 * Events are stored in (row, pattern, time) order at the exclusive prefix sum of outJumpCounts: outEventTimes (edge-length
 * units from the parent end) and outEventStates (the new state); *outEventCount receives their total.  Any output may be
 * NULL; only what is asked for is computed past the sampler and copied back.  Both event arrays NULL is the sizing query.
 * When events are asked for and their total exceeds eventCapacity, the event arrays are left untouched, *outEventCount and
 * every fixed-size output are written, and the call returns BEAGLE_ERROR_OUT_OF_RANGE; the draw is a pure function of the
 * arguments, so the call can be repeated with arrays of the right size.  No atomics: repeated calls are bit-identical.
 * Every other error returns before anything is launched (deferred work included) and leaves every output untouched:
 * BEAGLE_ERROR_OUT_OF_RANGE for whatever b200SampleAncestralStates rejects (its NULL-output rule aside), rateMatrix == NULL,
 * an entry of it not finite, a negative off-diagonal entry or a row sum larger in magnitude than 1e-9 mu,
 * categoryRatesIndex out of range, edgeLengths == NULL or an edgeLengths[r] (r >= 1) negative or not finite,
 * registerMatrices == NULL, registerCount outside 1..8, eventCapacity < 0, an event array without outEventCount;
 * BEAGLE_ERROR_NO_IMPLEMENTATION when mu tau_max > 700 (pi_0 would leave the normal range) or when S is so large that R and
 * two state vectors do not fit in one block's shared memory (S above 169 on an H100). */
BEAGLE_DLLEXPORT int b200SampleSubstitutionHistories(int instance, const int* nodeBuffers, const int* parentRows,
                                                     const int* matrixIndices, const double* edgeLengths, int count,
                                                     int rootBuffer, int categoryWeightsIndex, int stateFrequenciesIndex,
                                                     int categoryRatesIndex, const double* rateMatrix,
                                                     const double* registerMatrices, int registerCount,
                                                     unsigned long long seed, unsigned long long drawIndex, int* outStates,
                                                     int* outCategories, double* outBranchCounts, double* outPatternCounts,
                                                     int* outJumpCounts, long long eventCapacity, long long* outEventCount,
                                                     double* outEventTimes, int* outEventStates);
/* Host-logic test hook (no CUDA): the row rules of b200SampleAncestralStates for an instance with bufferCount buffers and
 * matrixCount matrices; 0 or BEAGLE_ERROR_OUT_OF_RANGE. */
BEAGLE_DLLEXPORT int b200DebugAncestralRows(const int* nodeBuffers, const int* parentRows, const int* matrixIndices, int count,
                                            int bufferCount, int matrixCount);

/* Host-logic test hook (no CUDA): the engine's execution plan for a 7-int-per-op list.  outOrder[n] = execution
 * position -> caller index; outSubs = (begin,end) position pairs of the independent subtree walks, grouped by phase;
 * outPhaseStart = index of each phase's first subtree (phases+1 entries); outCounts = {subtrees, phases}.
 * Array capacities: outSubs 2n ints, outPhaseStart n+1 ints.  preOrder: 0 = post-order list, 1 = pre-order list planned
 * as phased subtree walks of the out-forest, 2 = pre-order list planned as one launch per depth level. */
BEAGLE_DLLEXPORT int b200DebugPlan(const int* operations, int operationCount, int bufferCount, int fixedT, int wantSubs,
                                   int minT, int smallRemainder, int preOrder, int* outOrder, int* outSubs,
                                   int* outPhaseStart, int* outCounts);

/* Host-logic test hook (no CUDA): the post-order plan of a 7-int-per-op list (as b200DebugPlan with fixedT = 0), the
 * register forwarding between consecutive ops of a walk and the sibling-stack slots of the staged eigen walk.  Buffers
 * below tipCount are compact tips.  outRecords[5 * position] = {dest, child 1, child 2, flags, slots} of the op record
 * (a tip child is -(buffer + 1); flags bit 1 = child 1 is taken from registers; slots = byte 0 / 1 the slot child 1 / 2
 * is read from, byte 2 the slot the result is kept in, 0xFF = none); outSubs, outPhaseStart as in b200DebugPlan;
 * outCounts = {subtrees, phases, children read from a slot, internal children read from memory, deepest slot used}. */
BEAGLE_DLLEXPORT int b200DebugStackSlots(const int* operations, int operationCount, int bufferCount, int tipCount,
                                         int wantSubs, int minT, int smallRemainder, int* outRecords, int* outSubs,
                                         int* outPhaseStart, int* outCounts);

/* Host-logic test hook (no CUDA): the 4-state walk kernel of one phase of nSubs subtree walks over at most maxWindow
 * patterns, on an instance with the given padded categories (1, 2, 4, 8, 16 or 32), padded pattern count, SM count,
 * patterns per thread (1, 2 or 4), thin-phase rule and precision.  eigenForm: the list runs in eigen form; aligned: every
 * op covers all patterns; virt: the records name virtual cherries.  outRoute = {kernel, R, thin}; kernel 0 = matrix form,
 * 1 = eigen form with predicates, 2 = eigen form without, 3 = staged, 4 = staged with virtual cherries, 5 = no kernel. */
BEAGLE_DLLEXPORT int b200DebugWalkRoute(int matCP, int Ppad, int smCount, int walkR, int thinR1, int single, int nSubs,
                                        int maxWindow, int eigenForm, int aligned, int virt, int* outRoute);

#ifdef __cplusplus
}
#endif
#endif /* LIBHMSBEAGLE_B200_H */
