"""ctypes mirror of the Java binding in the reference's lib/beagle.jar.

``Beagle`` carries the same method names, argument order and meaning as the ``beagle.Beagle``
interface (42 methods, tests/golden/beagle_jar_abi.json); ``BeagleJNIImpl`` forwards each one 1:1
to the C ABI of our libhmsbeagle.so exactly as the jar's ``BeagleJNIImpl`` forwards to
``BeagleJNIWrapper`` natives, and raises ``BeagleException(functionName, errorCode)`` on a non-zero
return (``calculateRootLogLikelihoods`` lets -8 FLOATING_POINT through, as the jar does).
``BeagleFactory.loadBeagleInstance`` mirrors the factory the reference calls at
BeagleDataLikelihoodDelegate.java:439-452.

The product path is the CUDA library: if it is missing this module raises at load time -- there is
no Python/CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import numpy as np

NONE = -1
OPERATION_TUPLE_SIZE = 7
PARTITION_OPERATION_TUPLE_SIZE = 9

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class BeagleException(RuntimeError):
    def __init__(self, functionName: str, errCode: int):
        super().__init__(f"BEAGLE function, {functionName}, returned error code {errCode}")
        self.functionName = functionName
        self.errCode = errCode


class BeagleErrorCode:
    NO_ERROR = 0
    GENERAL_ERROR = -1
    OUT_OF_MEMORY_ERROR = -2
    UNIDENTIFIED_EXCEPTION_ERROR = -3
    UNINITIALIZED_INSTANCE_ERROR = -4
    OUT_OF_RANGE_ERROR = -5
    NO_RESOURCE_ERROR = -6
    NO_IMPLEMENTATION_ERROR = -7
    FLOATING_POINT_ERROR = -8


class BeagleFlag:
    PRECISION_SINGLE = 1 << 0
    PRECISION_DOUBLE = 1 << 1
    COMPUTATION_SYNCH = 1 << 2
    COMPUTATION_ASYNCH = 1 << 3
    EIGEN_REAL = 1 << 4
    EIGEN_COMPLEX = 1 << 5
    SCALING_MANUAL = 1 << 6
    SCALING_AUTO = 1 << 7
    SCALING_ALWAYS = 1 << 8
    SCALERS_RAW = 1 << 9
    SCALERS_LOG = 1 << 10
    VECTOR_SSE = 1 << 11
    VECTOR_NONE = 1 << 12
    THREADING_OPENMP = 1 << 13
    THREADING_NONE = 1 << 14
    PROCESSOR_CPU = 1 << 15
    PROCESSOR_GPU = 1 << 16
    SCALING_DYNAMIC = 1 << 19
    FRAMEWORK_CUDA = 1 << 22
    FRAMEWORK_OPENCL = 1 << 23
    FRAMEWORK_CPU = 1 << 27
    PARALLELOPS_STREAMS = 1 << 28
    PARALLELOPS_GRID = 1 << 29
    THREADING_CPP = 1 << 30
    PREORDER_TRANSPOSE_AUTO = 1 << 31
    VECTOR_TENSOR = 1 << 33


class _InstanceDetailsStruct(C.Structure):
    _fields_ = [("resourceNumber", C.c_int), ("resourceName", C.c_char_p), ("implName", C.c_char_p),
                ("implDescription", C.c_char_p), ("flags", C.c_long)]


class _ResourceStruct(C.Structure):
    _fields_ = [("name", C.c_char_p), ("description", C.c_char_p), ("supportFlags", C.c_long),
                ("requiredFlags", C.c_long)]


class _ResourceListStruct(C.Structure):
    _fields_ = [("list", C.POINTER(_ResourceStruct)), ("length", C.c_int)]


class InstanceDetails:
    def __init__(self, resourceNumber=0, flags=0, resourceName="", implementationName=""):
        self.resourceNumber = resourceNumber
        self.flags = flags
        self.resourceName = resourceName
        self.implementationName = implementationName

    def getFlags(self):
        return self.flags

    def getResourceNumber(self):
        return self.resourceNumber


class ResourceDetails:
    def __init__(self, number, name, description, flags):
        self.number, self.name, self.description, self.flags = number, name, description, flags


_I = C.c_int
_IP = C.POINTER(C.c_int)
_DP = C.POINTER(C.c_double)
_L = C.c_long

# name -> argtypes of every exported function of include/libhmsbeagle_b200.h (return type int unless noted)
_SIGNATURES = {
    "beagleGetVersion": ([], C.c_char_p),
    "beagleGetCitation": ([], C.c_char_p),
    "beagleGetResourceList": ([], C.POINTER(_ResourceListStruct)),
    "beagleGetBenchmarkedResourceList": ([_I, _I, _I, _I, _I, _IP, _I, _L, _L, _I, _I, _I, _L], C.c_void_p),
    "beagleCreateInstance": ([_I] * 9 + [_IP, _I, _L, _L, C.POINTER(_InstanceDetailsStruct)], _I),
    "beagleFinalizeInstance": ([_I], _I),
    "beagleFinalize": ([], _I),
    "beagleSetCPUThreadCount": ([_I, _I], _I),
    "beagleSetTipStates": ([_I, _I, _IP], _I),
    "beagleGetTipStates": ([_I, _I, _IP], _I),
    "beagleSetTipPartials": ([_I, _I, _DP], _I),
    "beagleSetPartials": ([_I, _I, _DP], _I),
    "beagleGetPartials": ([_I, _I, _I, _DP], _I),
    "beagleSetEigenDecomposition": ([_I, _I, _DP, _DP, _DP], _I),
    "beagleSetStateFrequencies": ([_I, _I, _DP], _I),
    "beagleSetCategoryWeights": ([_I, _I, _DP], _I),
    "beagleSetCategoryRates": ([_I, _DP], _I),
    "beagleSetCategoryRatesWithIndex": ([_I, _I, _DP], _I),
    "beagleSetPatternWeights": ([_I, _DP], _I),
    "beagleSetPatternPartitions": ([_I, _I, _IP], _I),
    "beagleUpdateTransitionMatrices": ([_I, _I, _IP, _IP, _IP, _DP, _I], _I),
    "beagleUpdateTransitionMatricesWithMultipleModels": ([_I, _IP, _IP, _IP, _IP, _IP, _DP, _I], _I),
    "beagleSetTransitionMatrix": ([_I, _I, _DP, C.c_double], _I),
    "beagleGetTransitionMatrix": ([_I, _I, _DP], _I),
    "beagleSetDifferentialMatrix": ([_I, _I, _DP], _I),
    "beagleConvolveTransitionMatrices": ([_I, _IP, _IP, _IP, _I], _I),
    "beagleAddTransitionMatrices": ([_I, _IP, _IP, _IP, _I], _I),
    "beagleTransposeTransitionMatrices": ([_I, _IP, _IP, _I], _I),
    "beagleUpdatePartials": ([_I, _IP, _I, _I], _I),
    "beagleUpdatePartialsByPartition": ([_I, _IP, _I], _I),
    "beagleWaitForPartials": ([_I, _IP, _I], _I),
    "beagleUpdatePrePartials": ([_I, _IP, _I, _I], _I),
    "beagleUpdatePrePartialsByPartition": ([_I, _IP, _I], _I),
    "beagleAccumulateScaleFactors": ([_I, _IP, _I, _I], _I),
    "beagleAccumulateScaleFactorsByPartition": ([_I, _IP, _I, _I, _I], _I),
    "beagleRemoveScaleFactors": ([_I, _IP, _I, _I], _I),
    "beagleRemoveScaleFactorsByPartition": ([_I, _IP, _I, _I, _I], _I),
    "beagleResetScaleFactors": ([_I, _I], _I),
    "beagleResetScaleFactorsByPartition": ([_I, _I, _I], _I),
    "beagleCopyScaleFactors": ([_I, _I, _I], _I),
    "beagleGetScaleFactors": ([_I, _I, _DP], _I),
    "beagleGetLogScaleFactors": ([_I, _I, _DP], _I),
    "beagleCalculateRootLogLikelihoods": ([_I, _IP, _IP, _IP, _IP, _I, _DP], _I),
    "beagleCalculateRootLogLikelihoodsByPartition": ([_I, _IP, _IP, _IP, _IP, _IP, _I, _I, _DP, _DP], _I),
    "beagleGetSiteLogLikelihoods": ([_I, _DP], _I),
    "beagleCalculateEdgeDerivatives": ([_I, _IP, _IP, _IP, _IP, _I, _DP, _DP, _DP], _I),
    "beagleCalculateCrossProductDerivative": ([_I, _IP, _IP, _IP, _IP, _DP, _I, _DP, _DP], _I),
    "b200SetKernelTiming": ([_I, _I], _I),
    "b200GetKernelTiming": ([_I, _I, _DP, C.POINTER(C.c_long)], _I),
    "b200CompressSitePatterns": ([_I, _I, _I, _IP, _DP, _IP, _IP, _DP, _IP], _I),
    "b200SampleAncestralStates": ([_I, _IP, _IP, _IP, _I, _I, _I, _I, C.c_ulonglong, C.c_ulonglong, _IP, _IP], _I),
    "b200DebugAncestralRows": ([_IP, _IP, _IP, _I, _I, _I], _I),
    "b200SampleMarkovJumps": ([_I, _IP, _IP, _IP, _DP, _I, _I, _I, _I, _I, _I, _DP, _I, C.c_ulonglong, C.c_ulonglong, _IP, _IP,
                               _DP, _DP], _I),
    "b200SampleSubstitutionHistories": ([_I, _IP, _IP, _IP, _DP, _I, _I, _I, _I, _I, _DP, _DP, _I, C.c_ulonglong,
                                         C.c_ulonglong, _IP, _IP, _DP, _DP, _IP, C.c_longlong, C.POINTER(C.c_longlong), _DP,
                                         _IP], _I),
    "b200GetSourceHash": ([], C.c_char_p),
    "b200GetFusedLaunches": ([_I], _L),
    "b200RootLogLikelihoodsByPartitionDevice": ([_I, _IP, _IP, _IP, _IP, _IP, _I, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)], _I),
    "b200SetShardDevices": ([_IP, _I], _I),
    "b200ExchangeConnectLocal": ([_IP, _I], _I),
    "b200ExchangeCreate": ([_I, _I, _I, C.c_void_p], _I),
    "b200ExchangeConnect": ([_I, C.c_void_p], _I),
    "b200HostAlloc": ([_L], C.c_void_p),
    "b200HostFree": ([C.c_void_p], None),
    "b200DebugPlan": ([_I if False else _IP, _I, _I, _I, _I, _I, _I, _I, _IP, _IP, _IP, _IP], _I),
    "b200DebugStackSlots": ([_IP, _I, _I, _I, _I, _I, _I, _IP, _IP, _IP, _IP], _I),
    "b200DebugWalkRoute": ([_I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _IP], _I),
    "b200RootLogLikelihoodDevice": ([_I, _I, _I, _I, _I, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)], _I),
}


def exported_symbols():
    return list(_SIGNATURES.keys())


def load_library(path: Optional[str] = None):
    """dlopen libhmsbeagle.so (built in-tree by build.py).  Raises if it is missing."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    path = path or os.environ.get("B200_BEAGLE_LIBRARY") or os.path.join(_HERE, "csrc", "libhmsbeagle.so")
    if not os.path.exists(path):
        raise FileNotFoundError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`; "
            "there is no CPU fallback for the product path")
    lib = C.CDLL(path)
    for name, (argtypes, restype) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = restype
    _LIB = lib
    return lib


def _ip(a):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(_IP)


def _dp(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_DP)


class Beagle:
    """Documentation-only statement of the ``beagle.Beagle`` interface (see BeagleJNIImpl)."""
    OPERATION_TUPLE_SIZE = OPERATION_TUPLE_SIZE
    PARTITION_OPERATION_TUPLE_SIZE = PARTITION_OPERATION_TUPLE_SIZE
    NONE = NONE


class BeagleJNIImpl(Beagle):
    """One engine instance; constructor arguments are those of the jar's BeagleJNIImpl.<init>."""

    def __init__(self, tipCount, partialsBufferCount, compactBufferCount, stateCount, patternCount,
                 eigenBufferCount, matrixBufferCount, categoryCount, scaleBufferCount,
                 resourceList: Optional[Sequence[int]], preferenceFlags: int, requirementFlags: int):
        self._lib = load_library()
        det = _InstanceDetailsStruct()
        rl = _ip(resourceList) if resourceList is not None else None
        inst = self._lib.beagleCreateInstance(tipCount, partialsBufferCount, compactBufferCount, stateCount,
                                              patternCount, eigenBufferCount, matrixBufferCount, categoryCount,
                                              scaleBufferCount, rl[1] if rl else None,
                                              len(resourceList) if resourceList is not None else 0,
                                              preferenceFlags, requirementFlags, C.byref(det))
        if inst < 0:
            raise BeagleException("create", inst)
        self.instance = inst
        self.patternCount = patternCount
        self.details = InstanceDetails(det.resourceNumber, det.flags,
                                       (det.resourceName or b"").decode(), (det.implName or b"").decode())

    def _check(self, name, rc):
        if rc != 0:
            raise BeagleException(name, rc)

    def getDetails(self):
        return self.details

    def finalize(self):
        if self.instance >= 0:
            rc = self._lib.beagleFinalizeInstance(self.instance)
            self.instance = -1
            self._check("finalize", rc)

    def setCPUThreadCount(self, threadCount):
        self._check("setCPUThreadCount", self._lib.beagleSetCPUThreadCount(self.instance, threadCount))

    def setPatternWeights(self, patternWeights):
        self._check("setPatternWeights", self._lib.beagleSetPatternWeights(self.instance, _dp(patternWeights)[1]))

    def setPatternPartitions(self, partitionCount, patternPartitions):
        self._check("setPatternPartitions",
                    self._lib.beagleSetPatternPartitions(self.instance, partitionCount, _ip(patternPartitions)[1]))

    def setTipStates(self, tipIndex, states):
        self._check("setTipStates", self._lib.beagleSetTipStates(self.instance, tipIndex, _ip(states)[1]))

    def getTipStates(self, tipIndex, states):
        self._check("getTipStates", self._lib.beagleGetTipStates(self.instance, tipIndex, states.ctypes.data_as(_IP)))

    def setTipPartials(self, tipIndex, partials):
        self._check("setTipPartials", self._lib.beagleSetTipPartials(self.instance, tipIndex, _dp(partials)[1]))

    def setPartials(self, bufferIndex, partials):
        self._check("setPartials", self._lib.beagleSetPartials(self.instance, bufferIndex, _dp(partials)[1]))

    def getPartials(self, bufferIndex, scaleIndex, outPartials):
        assert outPartials.dtype == np.float64 and outPartials.flags.c_contiguous
        self._check("getPartials", self._lib.beagleGetPartials(self.instance, bufferIndex, scaleIndex,
                                                               outPartials.ctypes.data_as(_DP)))

    def getLogScaleFactors(self, scaleIndex, outFactors):
        self._check("getLogScaleFactors", self._lib.beagleGetLogScaleFactors(self.instance, scaleIndex,
                                                                             outFactors.ctypes.data_as(_DP)))

    def getScaleFactors(self, scaleIndex, outFactors):
        self._check("getScaleFactors", self._lib.beagleGetScaleFactors(self.instance, scaleIndex,
                                                                       outFactors.ctypes.data_as(_DP)))

    def setEigenDecomposition(self, eigenIndex, eigenVectors, inverseEigenValues, eigenValues):
        self._check("setEigenDecomposition",
                    self._lib.beagleSetEigenDecomposition(self.instance, eigenIndex, _dp(eigenVectors)[1],
                                                          _dp(inverseEigenValues)[1], _dp(eigenValues)[1]))

    def setStateFrequencies(self, stateFrequenciesIndex, stateFrequencies):
        self._check("setStateFrequencies",
                    self._lib.beagleSetStateFrequencies(self.instance, stateFrequenciesIndex, _dp(stateFrequencies)[1]))

    def setCategoryWeights(self, categoryWeightsIndex, categoryWeights):
        self._check("setCategoryWeights",
                    self._lib.beagleSetCategoryWeights(self.instance, categoryWeightsIndex, _dp(categoryWeights)[1]))

    def setCategoryRates(self, inCategoryRates):
        self._check("setCategoryRates", self._lib.beagleSetCategoryRates(self.instance, _dp(inCategoryRates)[1]))

    def setCategoryRatesWithIndex(self, categoryRatesIndex, inCategoryRates):
        self._check("setCategoryRatesWithIndex",
                    self._lib.beagleSetCategoryRatesWithIndex(self.instance, categoryRatesIndex, _dp(inCategoryRates)[1]))

    def setTransitionMatrix(self, matrixIndex, inMatrix, paddedValue=0.0):
        self._check("setTransitionMatrix",
                    self._lib.beagleSetTransitionMatrix(self.instance, matrixIndex, _dp(inMatrix)[1], paddedValue))

    def getTransitionMatrix(self, matrixIndex, outMatrix):
        self._check("getTransitionMatrix",
                    self._lib.beagleGetTransitionMatrix(self.instance, matrixIndex, outMatrix.ctypes.data_as(_DP)))

    def updateTransitionMatrices(self, eigenIndex, probabilityIndices, firstDerivativeIndices,
                                 secondDerivativeIndices, edgeLengths, count):
        d1 = _ip(firstDerivativeIndices)
        d2 = _ip(secondDerivativeIndices)
        self._check("updateTransitionMatrices",
                    self._lib.beagleUpdateTransitionMatrices(self.instance, eigenIndex, _ip(probabilityIndices)[1],
                                                             d1[1] if d1 else None, d2[1] if d2 else None,
                                                             _dp(edgeLengths)[1], count))

    def updateTransitionMatricesWithMultipleModels(self, eigenIndices, categoryRateIndices, probabilityIndices,
                                                   firstDerivativeIndices, secondDerivativeIndices, edgeLengths, count):
        d1 = _ip(firstDerivativeIndices)
        d2 = _ip(secondDerivativeIndices)
        self._check("updateTransitionMatricesWithMultipleModels",
                    self._lib.beagleUpdateTransitionMatricesWithMultipleModels(
                        self.instance, _ip(eigenIndices)[1], _ip(categoryRateIndices)[1], _ip(probabilityIndices)[1],
                        d1[1] if d1 else None, d2[1] if d2 else None, _dp(edgeLengths)[1], count))

    def setDifferentialMatrix(self, matrixIndex, inMatrix):
        self._check("setDifferentialMatrix", self._lib.beagleSetDifferentialMatrix(self.instance, matrixIndex, _dp(inMatrix)[1]))

    def transposeTransitionMatrices(self, inputIndices, resultIndices, matrixCount):
        self._check("transposeTransitionMatrices",
                    self._lib.beagleTransposeTransitionMatrices(self.instance, _ip(inputIndices)[1], _ip(resultIndices)[1], matrixCount))

    def convolveTransitionMatrices(self, firstIndices, secondIndices, resultIndices, matrixCount):
        self._check("convolveTransitionMatrices",
                    self._lib.beagleConvolveTransitionMatrices(self.instance, _ip(firstIndices)[1], _ip(secondIndices)[1],
                                                               _ip(resultIndices)[1], matrixCount))

    def addTransitionMatrices(self, firstIndices, secondIndices, resultIndices, matrixCount):
        self._check("addTransitionMatrices",
                    self._lib.beagleAddTransitionMatrices(self.instance, _ip(firstIndices)[1], _ip(secondIndices)[1],
                                                          _ip(resultIndices)[1], matrixCount))

    def updatePrePartialsByPartition(self, operations, operationCount):
        self._check("updatePrePartialsByPartition",
                    self._lib.beagleUpdatePrePartialsByPartition(self.instance, _ip(operations)[1], operationCount))

    def updatePrePartials(self, operations, operationCount, cumulativeScaleIndex):
        self._check("updatePrePartials", self._lib.beagleUpdatePrePartials(self.instance, _ip(operations)[1],
                                                                           operationCount, cumulativeScaleIndex))

    def calculateEdgeDifferentials(self, postBufferIndices, preBufferIndices, derivativeMatrixIndices,
                                   categoryWeightsIndices, count, outDerivatives, outSumDerivatives,
                                   outSumSquaredDerivatives):
        ptr = lambda a: None if a is None else a.ctypes.data_as(_DP)
        self._check("calculateEdgeDifferentials",
                    self._lib.beagleCalculateEdgeDerivatives(self.instance, _ip(postBufferIndices)[1], _ip(preBufferIndices)[1],
                                                             _ip(derivativeMatrixIndices)[1], _ip(categoryWeightsIndices)[1],
                                                             count, ptr(outDerivatives), ptr(outSumDerivatives),
                                                             ptr(outSumSquaredDerivatives)))

    def calculateCrossProductDifferentials(self, postBufferIndices, preBufferIndices, categoryRatesIndices,
                                           categoryWeightsIndices, edgeLengths, count, outSumDerivatives,
                                           outSumSquaredDerivatives):
        ptr = lambda a: None if a is None else a.ctypes.data_as(_DP)
        lengths = np.ascontiguousarray(edgeLengths, dtype=np.float64)
        self._check("calculateCrossProductDifferentials",
                    self._lib.beagleCalculateCrossProductDerivative(
                        self.instance, _ip(postBufferIndices)[1], _ip(preBufferIndices)[1], _ip(categoryRatesIndices)[1],
                        _ip(categoryWeightsIndices)[1], lengths.ctypes.data_as(_DP), count, ptr(outSumDerivatives),
                        ptr(outSumSquaredDerivatives)))

    def updatePartials(self, operations, operationCount, cumulativeScaleIndex):
        self._check("updatePartials", self._lib.beagleUpdatePartials(self.instance, _ip(operations)[1],
                                                                     operationCount, cumulativeScaleIndex))

    def updatePartialsByPartition(self, operations, operationCount):
        self._check("updatePartialsByPartition",
                    self._lib.beagleUpdatePartialsByPartition(self.instance, _ip(operations)[1], operationCount))

    def waitForPartials(self, destinationPartials, destinationPartialsCount):
        self._check("waitForPartials", self._lib.beagleWaitForPartials(self.instance, _ip(destinationPartials)[1],
                                                                       destinationPartialsCount))

    def accumulateScaleFactors(self, scaleIndices, count, cumulativeScaleIndex):
        self._check("accumulateScaleFactors",
                    self._lib.beagleAccumulateScaleFactors(self.instance, _ip(scaleIndices)[1], count, cumulativeScaleIndex))

    def accumulateScaleFactorsByPartition(self, scaleIndices, count, cumulativeScaleIndex, partitionIndex):
        self._check("accumulateScaleFactorsByPartition",
                    self._lib.beagleAccumulateScaleFactorsByPartition(self.instance, _ip(scaleIndices)[1], count,
                                                                      cumulativeScaleIndex, partitionIndex))

    def removeScaleFactors(self, scaleIndices, count, cumulativeScaleIndex):
        self._check("removeScaleFactors",
                    self._lib.beagleRemoveScaleFactors(self.instance, _ip(scaleIndices)[1], count, cumulativeScaleIndex))

    def removeScaleFactorsByPartition(self, scaleIndices, count, cumulativeScaleIndex, partitionIndex):
        self._check("removeScaleFactorsByPartition",
                    self._lib.beagleRemoveScaleFactorsByPartition(self.instance, _ip(scaleIndices)[1], count,
                                                                  cumulativeScaleIndex, partitionIndex))

    def resetScaleFactors(self, cumulativeScaleIndex):
        self._check("resetScaleFactors", self._lib.beagleResetScaleFactors(self.instance, cumulativeScaleIndex))

    def resetScaleFactorsByPartition(self, cumulativeScaleIndex, partitionIndex):
        self._check("resetScaleFactorsByPartition",
                    self._lib.beagleResetScaleFactorsByPartition(self.instance, cumulativeScaleIndex, partitionIndex))

    def copyScaleFactors(self, destScalingIndex, srcScalingIndex):
        self._check("copyScaleFactors", self._lib.beagleCopyScaleFactors(self.instance, destScalingIndex, srcScalingIndex))

    def calculateRootLogLikelihoods(self, bufferIndices, categoryWeightsIndices, stateFrequenciesIndices,
                                    cumulativeScaleIndices, count, outSumLogLikelihood):
        rc = self._lib.beagleCalculateRootLogLikelihoods(self.instance, _ip(bufferIndices)[1],
                                                         _ip(categoryWeightsIndices)[1], _ip(stateFrequenciesIndices)[1],
                                                         _ip(cumulativeScaleIndices)[1], count,
                                                         outSumLogLikelihood.ctypes.data_as(_DP))
        # the jar swallows FLOATING_POINT_ERROR here (disassembly of BeagleJNIImpl.calculateRootLogLikelihoods)
        if rc != 0 and rc != BeagleErrorCode.FLOATING_POINT_ERROR:
            raise BeagleException("calculateRootLogLikelihoods", rc)

    def calculateRootLogLikelihoodsByPartition(self, bufferIndices, categoryWeightsIndices, stateFrequenciesIndices,
                                               cumulativeScaleIndices, partitionIndices, partitionCount, count,
                                               outSumLogLikelihoodByPartition, outSumLogLikelihood):
        rc = self._lib.beagleCalculateRootLogLikelihoodsByPartition(
            self.instance, _ip(bufferIndices)[1], _ip(categoryWeightsIndices)[1], _ip(stateFrequenciesIndices)[1],
            _ip(cumulativeScaleIndices)[1], _ip(partitionIndices)[1], partitionCount, count,
            outSumLogLikelihoodByPartition.ctypes.data_as(_DP), outSumLogLikelihood.ctypes.data_as(_DP))
        if rc != 0 and rc != BeagleErrorCode.FLOATING_POINT_ERROR:
            raise BeagleException("calculateRootLogLikelihoodsByPartition", rc)

    def getSiteLogLikelihoods(self, outLogLikelihoods):
        self._check("getSiteLogLikelihoods",
                    self._lib.beagleGetSiteLogLikelihoods(self.instance, outLogLikelihoods.ctypes.data_as(_DP)))

    # -- engine extensions used by bench.py ------------------------------------------------------
    def setKernelTiming(self, enable: bool):
        self._check("b200SetKernelTiming", self._lib.b200SetKernelTiming(self.instance, 1 if enable else 0))

    def getKernelTiming(self, which: int):
        ms = C.c_double(0.0)
        n = C.c_long(0)
        self._check("b200GetKernelTiming", self._lib.b200GetKernelTiming(self.instance, which, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def sampleAncestralStates(self, nodeBuffers, parentRows, matrixIndices, rootBuffer, categoryWeightsIndex,
                              stateFrequenciesIndex, seed, drawIndex):
        """One joint draw of ancestral states per pattern (b200SampleAncestralStates): rows in pre-order, row 0 the root ->
        (states int32 [rows][patternCount], categories int32 [patternCount])."""
        nb, pr, mi = _ip(nodeBuffers), _ip(parentRows), _ip(matrixIndices)
        count = len(nb[0])
        assert len(pr[0]) == count and len(mi[0]) == count
        states = np.zeros((count, self.patternCount), dtype=np.int32)
        cats = np.zeros(self.patternCount, dtype=np.int32)
        self._check("sampleAncestralStates",
                    self._lib.b200SampleAncestralStates(self.instance, nb[1], pr[1], mi[1], count, rootBuffer,
                                                        categoryWeightsIndex, stateFrequenciesIndex, seed, drawIndex,
                                                        states.ctypes.data_as(_IP), cats.ctypes.data_as(_IP)))
        return states, cats

    def sampleMarkovJumps(self, nodeBuffers, parentRows, matrixIndices, edgeLengths, rootBuffer, categoryWeightsIndex,
                          stateFrequenciesIndex, eigenIndex, categoryRatesIndex, registerMatrices, seed, drawIndex,
                          states=True, categories=True, branchCounts=True, patternCounts=True):
        """Markov-jump counts / rewards conditioned on one joint ancestral draw (b200SampleMarkovJumps): rows as in
        sampleAncestralStates, edgeLengths [rows], registerMatrices [registers][S][S] -> (states int32 [rows][patternCount],
        categories int32 [patternCount], branchCounts [registers][rows], patternCounts [registers][patternCount]); an output
        switched off by its flag is None and not copied back."""
        nb, pr, mi = _ip(nodeBuffers), _ip(parentRows), _ip(matrixIndices)
        count = len(nb[0])
        assert len(pr[0]) == count and len(mi[0]) == count
        lengths = _dp(np.asarray(edgeLengths, dtype=np.float64).reshape(count))
        regs = np.ascontiguousarray(registerMatrices, dtype=np.float64)
        G = regs.shape[0] if regs.ndim == 3 else 1
        regs = _dp(regs.reshape(-1))
        outs = (np.zeros((count, self.patternCount), dtype=np.int32) if states else None,
                np.zeros(self.patternCount, dtype=np.int32) if categories else None,
                np.zeros((G, count)) if branchCounts else None,
                np.zeros((G, self.patternCount)) if patternCounts else None)
        ptr = lambda a, t: None if a is None else a.ctypes.data_as(t)
        self._check("sampleMarkovJumps",
                    self._lib.b200SampleMarkovJumps(self.instance, nb[1], pr[1], mi[1], lengths[1], count, rootBuffer,
                                                    categoryWeightsIndex, stateFrequenciesIndex, eigenIndex,
                                                    categoryRatesIndex, regs[1], G, seed, drawIndex, ptr(outs[0], _IP),
                                                    ptr(outs[1], _IP), ptr(outs[2], _DP), ptr(outs[3], _DP)))
        return outs

    def sampleSubstitutionHistories(self, nodeBuffers, parentRows, matrixIndices, edgeLengths, rootBuffer,
                                    categoryWeightsIndex, stateFrequenciesIndex, categoryRatesIndex, rateMatrix,
                                    registerMatrices, seed, drawIndex, states=True, categories=True, branchCounts=True,
                                    patternCounts=True, jumpCounts=True, events=True):
        """Complete substitution histories by uniformization, conditioned on one joint ancestral draw
        (b200SampleSubstitutionHistories): rows and edgeLengths as in sampleMarkovJumps, rateMatrix [S][S] the generator Q,
        registerMatrices [registers][S][S] -> (states int32 [rows][patternCount], categories int32 [patternCount],
        branchCounts [registers][rows], patternCounts [registers][patternCount], jumpCounts int32 [rows][patternCount],
        eventTimes [events], eventStates int32 [events]); the events are in (row, pattern, time) order.  An output switched
        off by its flag is None and not copied back; with events, a sizing call first gives the arrays their length."""
        nb, pr, mi = _ip(nodeBuffers), _ip(parentRows), _ip(matrixIndices)
        count = len(nb[0])
        assert len(pr[0]) == count and len(mi[0]) == count
        lengths = _dp(np.asarray(edgeLengths, dtype=np.float64).reshape(count))
        Q = _dp(np.asarray(rateMatrix, dtype=np.float64).reshape(-1))
        regs = np.ascontiguousarray(registerMatrices, dtype=np.float64)
        G = regs.shape[0] if regs.ndim == 3 else 1
        regs = _dp(regs.reshape(-1))
        P = self.patternCount
        ptr = lambda a, t: None if a is None else a.ctypes.data_as(t)

        def call(outs, capacity, total, times, states_):
            return self._lib.b200SampleSubstitutionHistories(
                self.instance, nb[1], pr[1], mi[1], lengths[1], count, rootBuffer, categoryWeightsIndex,
                stateFrequenciesIndex, categoryRatesIndex, Q[1], regs[1], G, seed, drawIndex, ptr(outs[0], _IP),
                ptr(outs[1], _IP), ptr(outs[2], _DP), ptr(outs[3], _DP), ptr(outs[4], _IP), capacity, total,
                ptr(times, _DP), ptr(states_, _IP))

        total = C.c_longlong(0)
        times = eventStates = None
        if events:
            self._check("sampleSubstitutionHistories", call((None,) * 5, 0, C.byref(total), None, None))
            times, eventStates = np.zeros(total.value), np.zeros(total.value, dtype=np.int32)
        outs = (np.zeros((count, P), dtype=np.int32) if states else None,
                np.zeros(P, dtype=np.int32) if categories else None,
                np.zeros((G, count)) if branchCounts else None,
                np.zeros((G, P)) if patternCounts else None,
                np.zeros((count, P), dtype=np.int32) if jumpCounts else None)
        self._check("sampleSubstitutionHistories",
                    call(outs, total.value, C.byref(total) if events else None, times, eventStates))
        return outs + (times, eventStates)


class BeagleFactory:
    @staticmethod
    def getVersion() -> str:
        return load_library().beagleGetVersion().decode()

    @staticmethod
    def getResourceDetails():
        rl = load_library().beagleGetResourceList().contents
        return [ResourceDetails(i, rl.list[i].name.decode(), rl.list[i].description.decode(), rl.list[i].supportFlags)
                for i in range(rl.length)]

    @staticmethod
    def loadBeagleInstance(tipCount, partialsBufferCount, compactBufferCount, stateCount, patternCount,
                           eigenBufferCount, matrixBufferCount, categoryCount, scaleBufferCount,
                           resourceList, preferenceFlags, requirementFlags) -> BeagleJNIImpl:
        return BeagleJNIImpl(tipCount, partialsBufferCount, compactBufferCount, stateCount, patternCount,
                             eigenBufferCount, matrixBufferCount, categoryCount, scaleBufferCount,
                             resourceList, preferenceFlags, requirementFlags)


def compressSitePatterns(states, siteWeights=None, resource: int = 1):
    """SitePatterns (UNIQUE_ONLY) on the GPU: ``states`` int [taxa][sites] -> (patterns [taxa][P], weights [P],
    sitePatternIndices [sites]); see b200CompressSitePatterns in include/libhmsbeagle_b200.h."""
    lib = load_library()
    a = np.ascontiguousarray(states, dtype=np.int32)
    taxa, sites = a.shape
    idx = np.zeros(max(sites, 1), dtype=np.int32)
    pats = np.zeros(max(taxa * sites, 1), dtype=np.int32)
    w = np.zeros(max(sites, 1), dtype=np.float64)
    n = C.c_int(0)
    sw = None if siteWeights is None else np.ascontiguousarray(siteWeights, dtype=np.float64)
    rc = lib.b200CompressSitePatterns(resource, taxa, sites, a.ctypes.data_as(_IP),
                                      None if sw is None else sw.ctypes.data_as(_DP), idx.ctypes.data_as(_IP),
                                      pats.ctypes.data_as(_IP), w.ctypes.data_as(_DP), C.byref(n))
    if rc != 0:
        raise BeagleException("compressSitePatterns", rc)
    P = n.value
    return pats[:taxa * P].reshape(taxa, P).copy(), w[:P].copy(), idx[:sites].copy()


def checkAncestralRows(nodeBuffers, parentRows, matrixIndices, bufferCount, matrixCount) -> int:
    """The row rules of b200SampleAncestralStates on the host (b200DebugAncestralRows): 0 or OUT_OF_RANGE_ERROR."""
    lib = load_library()
    nb, pr, mi = _ip(nodeBuffers), _ip(parentRows), _ip(matrixIndices)
    return lib.b200DebugAncestralRows(nb[1], pr[1], mi[1], len(nb[0]), bufferCount, matrixCount)
