// multi.h -- entry points of the pattern-sharded instance (multi.cu) as api.cu forwards to them.
#pragma once
#include <functional>

namespace b200 {
struct Sharded;
int shSetTipStates(Sharded* sh, int tip, const int* states);
int shGetTipStates(Sharded* sh, int tip, int* states);
int shSetPartials(Sharded* sh, int buffer, const double* in, bool perCategory);
int shGetPartials(Sharded* sh, int buffer, int scaleIndex, double* out);
int shSetPatternWeights(Sharded* sh, const double* w);
int shBroadcast(Sharded* sh, const std::function<int(int)>& call);                       // call(child instance id)
int shGetPerPattern(Sharded* sh, double* out, const std::function<int(int, double*)>& call);
int shRoot(Sharded* sh, const int* bufferIndices, const int* wIdx, const int* fIdx, const int* cumIdx, int count, double* out);
int shEdgeDerivatives(Sharded* sh, const int* post, const int* pre, const int* dmat, const int* wIdx, int count, double* outPer,
                      double* outSum, double* outSumSq);
int shSampleAncestralStates(Sharded* sh, const int* nodeBuffers, const int* parentRows, const int* matrixIndices, int count,
                            int rootBuffer, int wIdx, int fIdx, unsigned long long seed, unsigned long long drawIndex,
                            int* outStates, int* outCategories);
int shSampleMarkovJumps(Sharded* sh, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                        const double* edgeLengths, int count, int rootBuffer, int wIdx, int fIdx, int eigenIndex, int rIdx,
                        const double* registerMatrices, int registerCount, unsigned long long seed, unsigned long long drawIndex,
                        int* outStates, int* outCategories, double* outBranchCounts, double* outPatternCounts);
int shSampleSubstitutionHistories(Sharded* sh, const int* nodeBuffers, const int* parentRows, const int* matrixIndices,
                                  const double* edgeLengths, int count, int rootBuffer, int wIdx, int fIdx, int rIdx,
                                  const double* rateMatrix, const double* registerMatrices, int registerCount,
                                  unsigned long long seed, unsigned long long drawIndex, int* outStates, int* outCategories,
                                  double* outBranchCounts, double* outPatternCounts, int* outJumpCounts, long long eventCapacity,
                                  long long* outEventCount, double* outEventTimes, int* outEventStates);
int shCrossProducts(Sharded* sh, const int* post, const int* pre, const int* rIdx, const int* wIdx, const double* lengths,
                    int count, double* outSum, double* outSumSq);
}  // namespace b200
