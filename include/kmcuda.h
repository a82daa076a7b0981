/*
 * kmcuda.h -- public C ABI of the H100-native libKMCUDA.
 *
 * This header re-states, declaration for declaration, the drop-in boundary of src-d/kmcuda
 * (reference: src/kmcuda.h).  Every enum value and every argument position crosses the ABI and is
 * therefore identical to the reference:
 *
 *   KMCUDAResult           reference src/kmcuda.h:41-54
 *   KMCUDAInitMethod       reference src/kmcuda.h:57-72
 *   KMCUDADistanceMetric   reference src/kmcuda.h:75-81
 *   kmeans_cuda()          reference src/kmcuda.h:118-123   (entry point in kmcuda_b200/csrc/api.cu)
 *   knn_cuda()             reference src/kmcuda.h:150-155   (entry point in kmcuda_b200/csrc/api.cu)
 *
 * Existing callers (the CPython module `libKMCUDA`, user C programs linking -lKMCUDA, ctypes/cgo
 * stubs -- see INTEGRATION.md) bind these two symbols and nothing else.  Shard-level entry points
 * for multi-process (one rank per GPU) integrations are declared separately in kmcuda_b200.h.
 */
#ifndef KMCUDA_KMCUDA_H
#define KMCUDA_KMCUDA_H

#include <stdint.h>

/* Error codes returned by every entry point (no exceptions cross the ABI). */
typedef enum {
  kmcudaSuccess = 0,                 /* all right */
  kmcudaInvalidArguments,            /* argument validation failed */
  kmcudaNoSuchDevice,                /* device mask names a GPU that does not exist */
  kmcudaMemoryAllocationFailure,     /* cudaMalloc failed */
  kmcudaRuntimeError,                /* a kernel launch / CUDA runtime call failed */
  kmcudaMemoryCopyError              /* a host<->device or peer copy failed */
} KMCUDAResult;

/* How the initial centroids are chosen. */
typedef enum {
  kmcudaInitMethodRandom = 0,        /* K distinct random samples */
  kmcudaInitMethodPlusPlus,          /* k-means++ */
  kmcudaInitMethodAFKMC2,            /* AFK-MC2; init_params -> uint32_t m (0 = 200) */
  kmcudaInitMethodImport             /* `centroids` holds the initial centroids on entry */
} KMCUDAInitMethod;

/* Distance between two points. */
typedef enum {
  kmcudaDistanceMetricL2,            /* Euclidean */
  kmcudaDistanceMetricCosine         /* angular; samples must be L2-normalised */
} KMCUDADistanceMetric;

#ifdef __cplusplus
extern "C" {
#endif

/*
 * K-means clustering (Lloyd, or Yinyang when yinyang_t*clusters_size >= 1 and tolerance < 0.11).
 *
 *  init, init_params  initialisation method (init_params: uint32_t* m for AFK-MC2, else ignored)
 *  tolerance          stop when reassignments <= tolerance * samples_size; in [0, 1]
 *  yinyang_t          groups = yinyang_t * clusters_size; in [0, 0.5]; 0 disables Yinyang
 *  metric             L2 or cosine
 *  samples_size       N  (>= clusters_size)
 *  features_size      D  (the number of half2 pairs when fp16x2 != 0)
 *  clusters_size      K  (>= 2, != UINT32_MAX)
 *  seed               srand() seed of the host RNG used by the init methods
 *  device             bit mask of GPUs, 0 = all
 *  device_ptrs        < 0: all pointers are host memory; >= 0: device memory on that GPU
 *  fp16x2             non-zero: data are half2, centroids are returned as half2
 *  verbosity          0 silent, 1 progress ("iteration %d: %u reassignments"), >= 2 debug
 *  samples            [N][D] row-major
 *  centroids          [K][D] row-major, output (input too with kmcudaInitMethodImport)
 *  assignments        [N] output
 *  average_distance   optional output, may be NULL
 */
KMCUDAResult kmeans_cuda(
    KMCUDAInitMethod init, const void *init_params, float tolerance, float yinyang_t,
    KMCUDADistanceMetric metric, uint32_t samples_size, uint16_t features_size,
    uint32_t clusters_size, uint32_t seed, uint32_t device, int32_t device_ptrs,
    int32_t fp16x2, int32_t verbosity, const float *samples, float *centroids,
    uint32_t *assignments, float *average_distance);

/*
 * Exact k nearest neighbours of every sample, accelerated by a precomputed clustering.
 *
 *  k                  neighbours per sample
 *  centroids          [K][D] input, assignments [N] input (a k-means result)
 *  neighbors          [N][k] output, ascending by distance, the sample itself excluded
 *  (other arguments as in kmeans_cuda)
 */
KMCUDAResult knn_cuda(
    uint16_t k, KMCUDADistanceMetric metric, uint32_t samples_size,
    uint16_t features_size, uint32_t clusters_size, uint32_t device,
    int32_t device_ptrs, int32_t fp16x2, int32_t verbosity,
    const float *samples, const float *centroids, const uint32_t *assignments,
    uint32_t *neighbors);

#ifdef __cplusplus
}  /* extern "C" */
#endif

#ifdef __cplusplus
#include <string>
#include <unordered_map>

namespace {
namespace kmcuda {
/* String -> enum tables used by language bindings (reference src/kmcuda.h:165-196). */
const std::unordered_map<std::string, KMCUDAInitMethod> init_methods{
    {"kmeans++", kmcudaInitMethodPlusPlus}, {"k-means++", kmcudaInitMethodPlusPlus},
    {"afkmc2", kmcudaInitMethodAFKMC2},     {"afk-mc2", kmcudaInitMethodAFKMC2},
    {"random", kmcudaInitMethodRandom}};

const std::unordered_map<std::string, KMCUDADistanceMetric> metrics{
    {"euclidean", kmcudaDistanceMetricL2},  {"L2", kmcudaDistanceMetricL2},
    {"l2", kmcudaDistanceMetricL2},         {"cos", kmcudaDistanceMetricCosine},
    {"cosine", kmcudaDistanceMetricCosine}, {"angular", kmcudaDistanceMetricCosine}};

const std::unordered_map<int, const char *> statuses{
    {kmcudaSuccess, "Success"},
    {kmcudaInvalidArguments, "InvalidArguments"},
    {kmcudaNoSuchDevice, "NoSuchDevice"},
    {kmcudaMemoryAllocationFailure, "MemoryAllocationFailure"},
    {kmcudaRuntimeError, "RuntimeError"},
    {kmcudaMemoryCopyError, "MemoryCopyError"}};
}  // namespace kmcuda
}  // namespace
#endif  /* __cplusplus */

#endif  /* KMCUDA_KMCUDA_H */
