// py_module.cc -- `import libKMCUDA`: the CPython face of the same shared object that exports the C ABI.
//
// Drop-in for the reference binding (reference src/python.cc): module name, function names, keyword
// names and defaults (python.cc:160-179, 413-426), ndarray / raw-device-pointer-tuple intake
// (:120-157, :232-278, :442-518), return types (:383-404, :619-631) and the error-code -> exception map
// (:365-381, :601-617) are the contract; the implementation is new.  The GIL is released around the
// library call (python.cc:357-363).
#define NPY_NO_DEPRECATED_API NPY_1_7_API_VERSION
#include <Python.h>
#include <numpy/arrayobject.h>

#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <string>

#include "kmcuda.h"
#include "kmcuda_b200.h"

namespace {

struct Ref {  // owned PyObject reference
  PyObject* p = nullptr;
  Ref() = default;
  explicit Ref(PyObject* o) : p(o) {}
  ~Ref() { Py_XDECREF(p); }
  Ref(const Ref&) = delete;
  Ref& operator=(const Ref&) = delete;
  void reset(PyObject* o) {
    Py_XDECREF(p);
    p = o;
  }
  PyArrayObject* arr() const { return reinterpret_cast<PyArrayObject*>(p); }
};

bool parse_metric(PyObject* obj, KMCUDADistanceMetric* metric) {
  if (obj == Py_None) {
    *metric = kmcudaDistanceMetricL2;
    return true;
  }
  if (!PyUnicode_Check(obj)) {
    PyErr_SetString(PyExc_TypeError, "\"metric\" must be either None or string.");
    return false;
  }
  const char* s = PyUnicode_AsUTF8(obj);
  auto it = s ? kmcuda::metrics.find(s) : kmcuda::metrics.end();
  if (it == kmcuda::metrics.end()) {
    PyErr_SetString(PyExc_ValueError, "Unknown metric. Supported values are \"L2\" and \"cos\".");
    return false;
  }
  *metric = it->second;
  return true;
}

// float16 2-D array -> fp16x2 mode (features halved), anything else is converted to float32
bool take_samples(PyObject* obj, Ref* keep, float** data, bool* fp16x2, uint32_t* n, uint32_t* d) {
  Ref probe(PyArray_FROM_O(obj));
  if (!probe.p) {
    PyErr_Clear();
    PyErr_SetString(PyExc_TypeError, "\"samples\" must be a 2D float32 or float16 numpy array");
    return false;
  }
  const bool half = PyArray_TYPE(probe.arr()) == NPY_FLOAT16;
  keep->reset(PyArray_FROM_OTF(obj, half ? NPY_FLOAT16 : NPY_FLOAT32, NPY_ARRAY_IN_ARRAY));
  if (!keep->p) {
    PyErr_Clear();
    PyErr_SetString(PyExc_TypeError, "\"samples\" must be a 2D float32 or float16 numpy array");
    return false;
  }
  if (PyArray_NDIM(keep->arr()) != 2) {
    PyErr_SetString(PyExc_ValueError, "\"samples\" must be a 2D numpy array");
    return false;
  }
  *n = static_cast<uint32_t>(PyArray_DIM(keep->arr(), 0));
  *d = static_cast<uint32_t>(PyArray_DIM(keep->arr(), 1));
  *fp16x2 = half;
  if (half) {
    if (*d % 2) {
      PyErr_SetString(PyExc_ValueError, "the number of features must be even in fp16 mode");
      return false;
    }
    *d /= 2;
  }
  *data = static_cast<float*>(PyArray_DATA(keep->arr()));
  return true;
}

bool check_features(uint32_t d) {
  if (d > UINT16_MAX) {
    PyErr_Format(PyExc_ValueError, "\"samples\": more than %" PRIu32 " features is not supported", d);
    return false;
  }
  return true;
}

PyObject* raise_for(int result, const char* fn) {
  switch (result) {
    case kmcudaInvalidArguments:
      PyErr_Format(PyExc_ValueError, "Invalid arguments were passed to %s", fn);
      break;
    case kmcudaNoSuchDevice:
      PyErr_SetString(PyExc_ValueError, "No such CUDA device exists");
      break;
    case kmcudaMemoryAllocationFailure:
      PyErr_SetString(PyExc_MemoryError, "Failed to allocate memory on GPU");
      break;
    case kmcudaMemoryCopyError:
      PyErr_SetString(PyExc_RuntimeError, "cudaMemcpy failed");
      break;
    case kmcudaRuntimeError:
      PyErr_Format(PyExc_AssertionError, "%s failure (bug?)", fn);
      break;
    default:
      PyErr_Format(PyExc_AssertionError, "Unknown error code returned from %s", fn);
  }
  return nullptr;
}

// the int members of the device-pointer tuples and of init=("afkmc2", m), Python ints or NumPy integers: false, with
// the Python error set, when `o` is not one or is out of range (negative, except for the device)
bool as_ull(PyObject* o, unsigned long long* out) {
  Ref i(PyNumber_Index(o));
  if (!i.p) return false;
  *out = PyLong_AsUnsignedLongLong(i.p);
  return !(*out == static_cast<unsigned long long>(-1) && PyErr_Occurred());
}

template <typename T>
bool as_pointer(PyObject* o, T** p) {
  unsigned long long v;
  if (!as_ull(o, &v)) return false;
  *p = reinterpret_cast<T*>(static_cast<uintptr_t>(v));
  return true;
}

bool as_u32(PyObject* o, uint32_t* out) {
  unsigned long long v;
  if (!as_ull(o, &v)) return false;
  *out = static_cast<uint32_t>(v);
  return true;
}

bool as_int(PyObject* o, int* out) {
  const long v = PyLong_AsLong(o);
  if (v == -1 && PyErr_Occurred()) return false;
  *out = static_cast<int>(v);
  return true;
}

// the shape member of a device-pointer samples tuple: (n, d) or (n, d, fp16x2)
bool take_shape(PyObject* shape, uint32_t* n, uint32_t* d, bool* fp16x2) {
  if (!PyTuple_Check(shape) || (PyTuple_GET_SIZE(shape) != 2 && PyTuple_GET_SIZE(shape) != 3)) {
    PyErr_SetString(PyExc_TypeError, "\"samples\"[2] must be a shape tuple");
    return false;
  }
  if (!as_u32(PyTuple_GET_ITEM(shape, 0), n) || !as_u32(PyTuple_GET_ITEM(shape, 1), d)) return false;
  if (PyTuple_GET_SIZE(shape) == 3) *fp16x2 = PyObject_IsTrue(PyTuple_GET_ITEM(shape, 2)) == 1;
  return true;
}

// sample_weight intake: with ndarray samples a 1-D numeric array-like of length n (converted to float32, kept alive in
// `keep`); with device-pointer samples an int device pointer on the samples' device
bool take_weights(PyObject* obj, bool device_samples, uint32_t n, Ref* keep, const float** data) {
  if (device_samples) {
    if (!PyLong_Check(obj) || PyBool_Check(obj)) {
      PyErr_SetString(PyExc_TypeError, "\"sample_weight\" must be a device pointer (integer) when \"samples\" is a "
                                       "pointer tuple");
      return false;
    }
    if (!as_pointer(obj, data)) return false;
    if (!*data) {
      PyErr_SetString(PyExc_ValueError, "\"sample_weight\" is null");
      return false;
    }
    return true;
  }
  Ref probe(PyArray_FROM_O(obj));
  if (!probe.p || !(PyArray_ISBOOL(probe.arr()) || PyArray_ISINTEGER(probe.arr()) || PyArray_ISFLOAT(probe.arr()))) {
    PyErr_Clear();
    PyErr_SetString(PyExc_TypeError, "\"sample_weight\" must be a 1D numeric array");
    return false;
  }
  if (PyArray_NDIM(probe.arr()) != 1) {
    PyErr_SetString(PyExc_ValueError, "\"sample_weight\" must be a 1D array");
    return false;
  }
  if (static_cast<uint64_t>(PyArray_DIM(probe.arr(), 0)) != n) {
    PyErr_SetString(PyExc_ValueError, "\"sample_weight\" must be of the same length as \"samples\"");
    return false;
  }
  keep->reset(PyArray_FROM_OTF(probe.p, NPY_FLOAT32, NPY_ARRAY_IN_ARRAY | NPY_ARRAY_FORCECAST));
  if (!keep->p) return false;
  *data = static_cast<const float*>(PyArray_DATA(keep->arr()));
  return true;
}

PyObject* build_kmeans_result(PyObject* centroids_arr, PyObject* assignments_arr, float* centroids,
                              uint32_t* assignments, int device_ptrs, int adflag, float average_distance,
                              bool want_inertia, double inertia);

PyObject* py_kmeans_cuda(PyObject*, PyObject* args, PyObject* kwargs) {
  long long clusters_arg = 0;   // range-checked below: "I" would wrap it modulo 2^32
  uint32_t afkmc2_m = 0, seed = static_cast<uint32_t>(time(nullptr)), device = 0;
  int32_t verbosity = 0;
  int adflag = 0;
  float tolerance = .01f, yinyang_t = .1f;
  PyObject *samples_obj, *init_obj = Py_None, *metric_obj = Py_None, *weight_obj = Py_None, *batch_obj = Py_None;
  PyObject *steps_obj = nullptr, *relocate_obj = Py_False, *n_init_obj = nullptr, *inertia_obj = Py_False;
  PyObject *bisecting_obj = Py_None, *max_iter_obj = nullptr, *tol_obj = Py_None, *n_iter_obj = Py_False;
  PyObject* init_size_obj = Py_None;
  static const char* kwlist[] = {"samples", "clusters", "tolerance", "init", "yinyang_t", "metric",
                                 "average_distance", "seed", "device", "verbosity", "sample_weight", "batch_size",
                                 "max_steps", "relocate_empty_clusters", "n_init", "inertia", "bisecting",
                                 "max_iter", "tol", "n_iter", "init_size", nullptr};
  if (!PyArg_ParseTupleAndKeywords(args, kwargs, "OL|fOfOpIIiOOOOOOOOOOO", const_cast<char**>(kwlist), &samples_obj,
                                   &clusters_arg, &tolerance, &init_obj, &yinyang_t, &metric_obj, &adflag, &seed,
                                   &device, &verbosity, &weight_obj, &batch_obj, &steps_obj, &relocate_obj,
                                   &n_init_obj, &inertia_obj, &bisecting_obj, &max_iter_obj, &tol_obj, &n_iter_obj,
                                   &init_size_obj))
    return nullptr;
  // bisecting k-means (kmcuda_b200.h, kmcuda_b200_kmeans_bisecting): None or a strategy name
  int32_t strategy = -1;
  if (bisecting_obj != Py_None) {
    if (!PyUnicode_Check(bisecting_obj)) {
      PyErr_SetString(PyExc_TypeError, "\"bisecting\" must be None or a string");
      return nullptr;
    }
    const char* b = PyUnicode_AsUTF8(bisecting_obj);
    if (b && strcmp(b, "biggest_inertia") == 0) strategy = 0;
    else if (b && strcmp(b, "largest_cluster") == 0) strategy = 1;
    else {
      PyErr_Clear();
      PyErr_SetString(PyExc_ValueError, "\"bisecting\" must be \"biggest_inertia\" or \"largest_cluster\"");
      return nullptr;
    }
  }
  // relocation of empty clusters (kmcuda_b200.h, kmcuda_b200_kmeans_relocate): a bool, not with mini-batch
  if (!(PyBool_Check(relocate_obj) || PyArray_IsScalar(relocate_obj, Bool))) {
    PyErr_SetString(PyExc_TypeError, "\"relocate_empty_clusters\" must be a bool");
    return nullptr;
  }
  const bool relocate = PyObject_IsTrue(relocate_obj) == 1;
  // mini-batch k-means (kmcuda_b200.h): batch_size an integer >= 1, max_steps an integer >= 0
  uint32_t batch_size = 0, max_steps = 0;
  auto take_count = [](PyObject* o, const char* name, unsigned long lo, uint32_t* out) {
    if (PyBool_Check(o) || !(PyLong_Check(o) || PyArray_IsScalar(o, Integer))) {
      PyErr_Format(PyExc_TypeError, "\"%s\" must be an integer", name);
      return false;
    }
    int overflow = 0;
    const long long v = PyLong_AsLongLongAndOverflow(o, &overflow);
    if (overflow || v < static_cast<long long>(lo) || v > 0xFFFFFFFFll) {
      PyErr_Clear();
      PyErr_Format(PyExc_ValueError, "\"%s\" must be an integer in [%lu, 2^32)", name, lo);
      return false;
    }
    *out = static_cast<uint32_t>(v);
    return true;
  };
  if (batch_obj != Py_None && !take_count(batch_obj, "batch_size", 1, &batch_size)) return nullptr;
  if (steps_obj && !take_count(steps_obj, "max_steps", 0, &max_steps)) return nullptr;
  if (max_steps && !batch_size) {
    PyErr_SetString(PyExc_ValueError, "\"max_steps\" applies to mini-batch runs only: pass \"batch_size\" too");
    return nullptr;
  }
  if (relocate && batch_obj != Py_None) {
    PyErr_SetString(PyExc_ValueError, "\"relocate_empty_clusters\" applies to Lloyd / Yinyang runs: mini-batch "
                                      "k-means (\"batch_size\") reassigns its clusters itself");
    return nullptr;
  }
  if (strategy >= 0) {
    // "random", "greedy-k-means++" / "greedy-kmeans++", or a tuple whose first item is a greedy name
    PyObject* name = init_obj;
    const bool tuple = init_obj && PyTuple_Check(init_obj);
    if (tuple) name = PyTuple_Size(init_obj) > 0 ? PyTuple_GetItem(init_obj, 0) : nullptr;
    const char* i = name && PyUnicode_Check(name) ? PyUnicode_AsUTF8(name) : nullptr;
    const bool greedy_name = i && (strcmp(i, "greedy-k-means++") == 0 || strcmp(i, "greedy-kmeans++") == 0);
    if (batch_obj != Py_None || max_steps || relocate) {
      PyErr_SetString(PyExc_ValueError, "\"bisecting\" cannot be combined with \"batch_size\", \"max_steps\" or "
                                        "\"relocate_empty_clusters\"");
      return nullptr;
    }
    if (!(greedy_name || (!tuple && i && strcmp(i, "random") == 0))) {
      PyErr_Clear();
      PyErr_SetString(PyExc_ValueError,
                      "\"bisecting\" takes init=\"random\", \"greedy-k-means++\" or (\"greedy-k-means++\", L)");
      return nullptr;
    }
  }
  // scikit-learn's stopping rule (kmcuda_b200.h, kmcuda_b200_kmeans_center_shift): tol None or a real number >= 0,
  // n_iter a bool that needs tol; not with mini-batch or bisecting
  const bool center_shift = tol_obj != Py_None;
  double tol = 0;
  if (center_shift) {
    if (PyBool_Check(tol_obj) || PyArray_IsScalar(tol_obj, Bool) ||
        !(PyFloat_Check(tol_obj) || PyLong_Check(tol_obj) || PyArray_IsScalar(tol_obj, Floating) ||
          PyArray_IsScalar(tol_obj, Integer))) {
      PyErr_SetString(PyExc_TypeError, "\"tol\" must be None or a real number");
      return nullptr;
    }
    tol = PyFloat_AsDouble(tol_obj);
    if (PyErr_Occurred()) return nullptr;
    if (!(std::isfinite(tol) && tol >= 0)) {
      PyErr_SetString(PyExc_ValueError, "\"tol\" must be a finite number >= 0");
      return nullptr;
    }
    if (batch_obj != Py_None || strategy >= 0) {
      PyErr_SetString(PyExc_ValueError, "\"tol\" applies to Lloyd / Yinyang runs: mini-batch (\"batch_size\") and "
                                        "bisecting runs scale \"tolerance\" themselves");
      return nullptr;
    }
  }
  if (!(PyBool_Check(n_iter_obj) || PyArray_IsScalar(n_iter_obj, Bool))) {
    PyErr_SetString(PyExc_TypeError, "\"n_iter\" must be a bool");
    return nullptr;
  }
  const bool want_n_iter = PyObject_IsTrue(n_iter_obj) == 1;
  if (want_n_iter && !center_shift) {
    PyErr_SetString(PyExc_ValueError, "\"n_iter\" needs \"tol\": only runs with scikit-learn's stopping rule count "
                                      "iterations");
    return nullptr;
  }
  uint32_t max_iter = 0;
  if (max_iter_obj && !take_count(max_iter_obj, "max_iter", 0, &max_iter)) return nullptr;
  if (max_iter && strategy < 0 && !center_shift) {
    PyErr_SetString(PyExc_ValueError, "\"max_iter\" applies to bisecting runs and runs with \"tol\" only: pass one "
                                      "of them too");
    return nullptr;
  }
  // the init stage of mini-batch k-means (kmcuda_b200.h, kmcuda_b200_kmeans_minibatch_init): init_size None (seed on
  // all rows), an integer >= 1 or "auto"; with batch_size only
  uint32_t init_size = 0;
  if (init_size_obj != Py_None) {
    if (PyUnicode_Check(init_size_obj)) {
      const char* a = PyUnicode_AsUTF8(init_size_obj);
      if (!a || strcmp(a, "auto") != 0) {
        PyErr_Clear();
        PyErr_SetString(PyExc_ValueError, "\"init_size\" must be None, an integer >= 1 or \"auto\"");
        return nullptr;
      }
      init_size = KMCUDA_B200_INIT_SIZE_AUTO;
    } else {
      if (PyBool_Check(init_size_obj) || !(PyLong_Check(init_size_obj) || PyArray_IsScalar(init_size_obj, Integer))) {
        PyErr_SetString(PyExc_TypeError, "\"init_size\" must be None, an integer or \"auto\"");
        return nullptr;
      }
      int overflow = 0;
      const long long v = PyLong_AsLongLongAndOverflow(init_size_obj, &overflow);
      if ((v == -1 && PyErr_Occurred()) || overflow < 0 || (!overflow && v < 1)) {
        PyErr_Clear();
        PyErr_SetString(PyExc_ValueError, "\"init_size\" must be None, an integer >= 1 or \"auto\"");
        return nullptr;
      }
      // every size from the number of rows up seeds on all rows; the largest value is the "auto" constant
      init_size = overflow || v >= KMCUDA_B200_INIT_SIZE_AUTO ? KMCUDA_B200_INIT_SIZE_AUTO - 1
                                                              : static_cast<uint32_t>(v);
    }
    if (strategy >= 0 || batch_obj == Py_None) {
      PyErr_SetString(PyExc_ValueError, "\"init_size\" applies to mini-batch runs only: pass \"batch_size\" and no "
                                        "\"bisecting\"");
      return nullptr;
    }
  }
  // restarts (kmcuda_b200.h, kmcuda_b200_kmeans_restarts): n_init an integer >= 1, inertia a bool; with mini-batch
  // n_init needs init_size (it is the number of inits ranked on a validation batch)
  uint32_t n_init = 1;
  if (n_init_obj && !take_count(n_init_obj, "n_init", 1, &n_init)) return nullptr;
  if (!(PyBool_Check(inertia_obj) || PyArray_IsScalar(inertia_obj, Bool))) {
    PyErr_SetString(PyExc_TypeError, "\"inertia\" must be a bool");
    return nullptr;
  }
  const bool want_inertia = PyObject_IsTrue(inertia_obj) == 1;
  if ((n_init != 1 && !init_size) && batch_obj != Py_None) {
    PyErr_SetString(PyExc_ValueError, "\"n_init\" > 1 with mini-batch k-means (\"batch_size\") needs \"init_size\": "
                                      "the inits are ranked on a validation batch of that many rows");
    return nullptr;
  }
  if (want_inertia && batch_obj != Py_None) {
    PyErr_SetString(PyExc_ValueError, "\"inertia\" applies to Lloyd / Yinyang and bisecting runs, not to mini-batch "
                                      "k-means (\"batch_size\")");
    return nullptr;
  }
  KMCUDAInitMethod init = kmcudaInitMethodPlusPlus;
  auto named_init = [&init](PyObject* o) {
    const char* s = PyUnicode_Check(o) ? PyUnicode_AsUTF8(o) : nullptr;
    if (s && (strcmp(s, "k-means||") == 0 || strcmp(s, "kmeans||") == 0)) {   // kmcuda_b200.h, not in kmcuda.h's table
      init = kmcudaInitMethodKMeansParallel;
      return true;
    }
    if (s && (strcmp(s, "greedy-k-means++") == 0 || strcmp(s, "greedy-kmeans++") == 0)) {   // kmcuda_b200.h too
      init = kmcudaInitMethodGreedyPlusPlus;
      return true;
    }
    auto it = s ? kmcuda::init_methods.find(s) : kmcuda::init_methods.end();
    if (it == kmcuda::init_methods.end()) {
      PyErr_SetString(PyExc_ValueError, "Unknown centroids initialization method. Supported values are "
                                        "\"kmeans++\", \"random\" and <numpy array>.");
      return false;
    }
    init = it->second;
    return true;
  };
  if (init_obj == Py_None) {
    init = kmcudaInitMethodPlusPlus;
  } else if (PyUnicode_Check(init_obj)) {
    if (!named_init(init_obj)) return nullptr;
  } else if (PyTuple_Check(init_obj)) {
    PyObject* first = PyTuple_Size(init_obj) > 0 ? PyTuple_GetItem(init_obj, 0) : nullptr;
    if (!first || first == Py_None) {
      PyErr_SetString(PyExc_ValueError, "centroid initialization method may not be null.");
      return nullptr;
    }
    if (!named_init(first)) return nullptr;
    if (PyTuple_Size(init_obj) > 1 && init == kmcudaInitMethodAFKMC2 &&
        !as_u32(PyTuple_GetItem(init_obj, 1), &afkmc2_m))
      return nullptr;
    const bool greedy = init == kmcudaInitMethodGreedyPlusPlus;
    if (PyTuple_Size(init_obj) > 1 && (init == kmcudaInitMethodKMeansParallel || greedy)) {
      // k-means|| rounds or greedy k-means++ trials: an integer in [0, 32]
      PyObject* r = PyTuple_GetItem(init_obj, 1);
      long v = -1;
      if (PyLong_Check(r) && !PyBool_Check(r)) {
        int overflow = 0;
        v = PyLong_AsLongAndOverflow(r, &overflow);
        if (overflow) v = -1;
      } else if (PyArray_IsScalar(r, Integer)) {
        v = PyLong_AsLong(r);
      }
      if (v < 0 || v > 32) {
        PyErr_Clear();
        PyErr_SetString(PyExc_ValueError, greedy ? "greedy k-means++ trials must be an integer in [0, 32]"
                                                 : "k-means|| rounds must be an integer in [0, 32]");
        return nullptr;
      }
      afkmc2_m = static_cast<uint32_t>(v);
    }
  } else {
    init = kmcudaInitMethodImport;
  }
  if (init == kmcudaInitMethodImport && n_init > 1) {
    PyErr_SetString(PyExc_ValueError, "\"n_init\" > 1 needs a seeding method: with imported centroids every restart "
                                      "is the same run");
    return nullptr;
  }
  if (init == kmcudaInitMethodImport && init_size) {
    PyErr_SetString(PyExc_ValueError, "\"init_size\" needs a seeding method: imported centroids read no rows");
    return nullptr;
  }
  KMCUDADistanceMetric metric;
  if (!parse_metric(metric_obj, &metric)) return nullptr;
  if (clusters_arg < 2 || clusters_arg >= UINT32_MAX) {
    PyErr_SetString(PyExc_ValueError, "\"clusters\" must be greater than 1 and less than (1 << 32) - 1");
    return nullptr;
  }
  const uint32_t clusters = static_cast<uint32_t>(clusters_arg);
  if (init_size && init_size != KMCUDA_B200_INIT_SIZE_AUTO && init_size < clusters) {
    PyErr_SetString(PyExc_ValueError, "\"init_size\" must be at least the number of clusters");
    return nullptr;
  }
  float *samples = nullptr, *centroids = nullptr;
  uint32_t* assignments = nullptr;
  uint32_t n = 0, d = 0;
  int device_ptrs = -1;
  bool fp16x2 = false;
  Ref keep_samples;
  if (PyTuple_Check(samples_obj)) {
    const Py_ssize_t size = PyTuple_GET_SIZE(samples_obj);
    if (size != 3 && size != 5) {
      PyErr_SetString(PyExc_ValueError, "len(\"samples\") must be either 3 or 5");
      return nullptr;
    }
    PyObject* ptr = PyTuple_GET_ITEM(samples_obj, 0);
    if (!PyLong_Check(ptr)) {
      PyErr_SetString(PyExc_ValueError, "\"samples\"[0] is not a pointer (integer)");
      return nullptr;
    }
    if (!as_pointer(ptr, &samples)) return nullptr;
    if (!samples) {
      PyErr_SetString(PyExc_ValueError, "\"samples\"[0] is null");
      return nullptr;
    }
    if (!as_int(PyTuple_GET_ITEM(samples_obj, 1), &device_ptrs)) return nullptr;
    if (!take_shape(PyTuple_GET_ITEM(samples_obj, 2), &n, &d, &fp16x2)) return nullptr;
    if (size == 5 && (!as_pointer(PyTuple_GET_ITEM(samples_obj, 3), &centroids) ||
                      !as_pointer(PyTuple_GET_ITEM(samples_obj, 4), &assignments)))
      return nullptr;
  } else if (!take_samples(samples_obj, &keep_samples, &samples, &fp16x2, &n, &d)) {
    return nullptr;
  }
  if (!check_features(d)) return nullptr;
  const float* weights = nullptr;
  Ref keep_weights;
  if (weight_obj != Py_None && !take_weights(weight_obj, device_ptrs >= 0, n, &keep_weights, &weights)) return nullptr;
  Ref centroids_arr, assignments_arr;
  if (device_ptrs < 0) {
    npy_intp cdims[2] = {static_cast<npy_intp>(clusters), static_cast<npy_intp>(fp16x2 ? d * 2 : d)};
    centroids_arr.reset(PyArray_EMPTY(2, cdims, fp16x2 ? NPY_FLOAT16 : NPY_FLOAT32, 0));
    npy_intp adims[1] = {static_cast<npy_intp>(n)};
    assignments_arr.reset(PyArray_EMPTY(1, adims, NPY_UINT32, 0));
    if (!centroids_arr.p || !assignments_arr.p) return nullptr;
    centroids = static_cast<float*>(PyArray_DATA(centroids_arr.arr()));
    assignments = static_cast<uint32_t*>(PyArray_DATA(assignments_arr.arr()));
  } else if (!centroids) {
    // outputs are allocated on the caller's device and handed over as raw pointers (python.cc:298-313)
    void *c = nullptr, *a = nullptr;
    int rc = kmcuda_b200_device_malloc(device_ptrs, static_cast<uint64_t>(clusters) * d * sizeof(float), &c);
    if (rc == kmcudaSuccess) rc = kmcuda_b200_device_malloc(device_ptrs, static_cast<uint64_t>(n) * 4, &a);
    if (rc != kmcudaSuccess) return raise_for(rc, "kmeans_cuda");
    centroids = static_cast<float*>(c);
    assignments = static_cast<uint32_t*>(a);
  }
  if (init == kmcudaInitMethodImport) {
    Ref imp(PyArray_FROM_OTF(init_obj, NPY_FLOAT32, NPY_ARRAY_IN_ARRAY));
    if (!imp.p) {
      PyErr_Clear();
      PyErr_SetString(PyExc_TypeError, "\"init\" centroids must be a 2D numpy array");
      return nullptr;
    }
    if (PyArray_NDIM(imp.arr()) != 2) {
      PyErr_SetString(PyExc_ValueError, "\"init\" centroids must be a 2D numpy array");
      return nullptr;
    }
    if (static_cast<uint32_t>(PyArray_DIM(imp.arr(), 0)) != clusters) {
      PyErr_SetString(PyExc_ValueError, "\"init\" centroids shape[0] does not match the number of clusters");
      return nullptr;
    }
    if (static_cast<uint32_t>(PyArray_DIM(imp.arr(), 1)) != d) {
      PyErr_SetString(PyExc_ValueError, "\"init\" centroids shape[1] does not match the number of features");
      return nullptr;
    }
    const size_t bytes = static_cast<size_t>(clusters) * d * sizeof(float);
    if (device_ptrs < 0) {
      memcpy(centroids, PyArray_DATA(imp.arr()), bytes);
    } else {
      int rc = kmcuda_b200_device_memcpy(device_ptrs, centroids, PyArray_DATA(imp.arr()), bytes, 1);
      if (rc != kmcudaSuccess) return raise_for(rc, "kmeans_cuda");
    }
  }
  float average_distance = 0;
  double inertia = 0;
  uint32_t n_iter = 0;
  int result;
  if ((batch_size || strategy >= 0) && yinyang_t > 0 && verbosity > 0) {
    printf("%s k-means: yinyang_t is ignored\n", batch_size ? "mini-batch" : "bisecting");
    fflush(stdout);
  }
  float* const avg = adflag ? &average_distance : nullptr;
  double* const inertia_out = want_inertia ? &inertia : nullptr;
  const uint16_t features = static_cast<uint16_t>(d);
  Py_BEGIN_ALLOW_THREADS
  if (center_shift)
    result = kmcuda_b200_kmeans_center_shift(init, &afkmc2_m, static_cast<float>(tol), yinyang_t, metric, n, features,
                                             clusters, seed, device, device_ptrs, fp16x2, verbosity, samples, weights,
                                             relocate ? 1 : 0, n_init, max_iter, centroids, assignments, avg,
                                             inertia_out, want_n_iter ? &n_iter : nullptr);
  else if (strategy >= 0)
    result = kmcuda_b200_kmeans_bisecting(init, &afkmc2_m, tolerance, metric, n, features, clusters, seed, device,
                                          device_ptrs, fp16x2, verbosity, samples, weights, strategy, n_init, max_iter,
                                          centroids, assignments, avg, inertia_out);
  else if (batch_size)   // init_size 0 and n_init 1: the documented equal of kmcuda_b200_kmeans_minibatch()
    result = kmcuda_b200_kmeans_minibatch_init(init, &afkmc2_m, tolerance, metric, n, features, clusters, seed, device,
                                               device_ptrs, fp16x2, verbosity, samples, weights, batch_size, max_steps,
                                               init_size, n_init, centroids, assignments, avg);
  else   // Lloyd / Yinyang with any weights, relocation and n_init: with n_init 1 and no inertia the header documents
         // this call as bit-identical to kmeans_cuda(), _weighted() and _relocate()
    result = kmcuda_b200_kmeans_restarts(init, &afkmc2_m, tolerance, yinyang_t, metric, n, features, clusters, seed,
                                         device, device_ptrs, fp16x2, verbosity, samples, weights, relocate ? 1 : 0,
                                         n_init, centroids, assignments, avg, inertia_out);
  Py_END_ALLOW_THREADS
  if (result != kmcudaSuccess) return raise_for(result, "kmeans_cuda");
  if (want_n_iter) {   // the result below with the iteration count appended
    Ref head(build_kmeans_result(centroids_arr.p, assignments_arr.p, centroids, assignments, device_ptrs, adflag,
                                 average_distance, want_inertia, inertia));
    Ref tail(Py_BuildValue("(k)", static_cast<unsigned long>(n_iter)));
    if (!head.p || !tail.p) return nullptr;
    return PySequence_Concat(head.p, tail.p);
  }
  return build_kmeans_result(centroids_arr.p, assignments_arr.p, centroids, assignments, device_ptrs, adflag,
                             average_distance, want_inertia, inertia);
}

// (centroids, assignments[, avg][, inertia]): arrays for host samples, raw device pointers for device samples
PyObject* build_kmeans_result(PyObject* centroids_arr, PyObject* assignments_arr, float* centroids,
                              uint32_t* assignments, int device_ptrs, int adflag, float average_distance,
                              bool want_inertia, double inertia) {
  if (want_inertia) {
    if (device_ptrs < 0) {
      if (!adflag) return Py_BuildValue("OOd", centroids_arr, assignments_arr, inertia);
      return Py_BuildValue("OOfd", centroids_arr, assignments_arr, average_distance, inertia);
    }
    const unsigned long long cp = reinterpret_cast<uintptr_t>(centroids), ap = reinterpret_cast<uintptr_t>(assignments);
    if (!adflag) return Py_BuildValue("KKd", cp, ap, inertia);
    return Py_BuildValue("KKfd", cp, ap, average_distance, inertia);
  }
  if (device_ptrs < 0) {
    if (!adflag) return Py_BuildValue("OO", centroids_arr, assignments_arr);
    return Py_BuildValue("OOf", centroids_arr, assignments_arr, average_distance);
  }
  const unsigned long long cp = reinterpret_cast<uintptr_t>(centroids), ap = reinterpret_cast<uintptr_t>(assignments);
  if (!adflag) return Py_BuildValue("KK", cp, ap);
  return Py_BuildValue("KKf", cp, ap, average_distance);
}

PyObject* py_knn_cuda(PyObject*, PyObject* args, PyObject* kwargs) {
  uint32_t device = 0;
  long long k = 0;   // range-checked below: "I" would wrap it modulo 2^32
  int32_t verbosity = 0;
  PyObject *samples_obj, *centroids_obj, *assignments_obj, *metric_obj = Py_None;
  static const char* kwlist[] = {"k", "samples", "centroids", "assignments", "metric", "device", "verbosity", nullptr};
  if (!PyArg_ParseTupleAndKeywords(args, kwargs, "LOOO|OIi", const_cast<char**>(kwlist), &k, &samples_obj,
                                   &centroids_obj, &assignments_obj, &metric_obj, &device, &verbosity))
    return nullptr;
  KMCUDADistanceMetric metric;
  if (!parse_metric(metric_obj, &metric)) return nullptr;
  if (k <= 0 || k > UINT16_MAX) {
    PyErr_SetString(PyExc_ValueError, "\"k\" must be greater than 0 and less than (1 << 16)");
    return nullptr;
  }
  float *samples = nullptr, *centroids = nullptr;
  uint32_t *assignments = nullptr, *neighbors = nullptr;
  uint32_t n = 0, d = 0, clusters = 0;
  int device_ptrs = -1;
  bool fp16x2 = false;
  Ref keep_s, keep_c, keep_a, neighbors_arr;
  if (PyTuple_Check(samples_obj)) {
    if (PyTuple_GET_SIZE(samples_obj) != 3) {
      PyErr_SetString(PyExc_ValueError, "len(\"samples\") must be 3");
      return nullptr;
    }
    if (!PyTuple_Check(centroids_obj) || PyTuple_GET_SIZE(centroids_obj) != 2) {
      PyErr_SetString(PyExc_ValueError, "\"centroids\" must be a tuple of length 2");
      return nullptr;
    }
    if (!as_pointer(PyTuple_GET_ITEM(samples_obj, 0), &samples) ||
        !as_int(PyTuple_GET_ITEM(samples_obj, 1), &device_ptrs) ||
        !take_shape(PyTuple_GET_ITEM(samples_obj, 2), &n, &d, &fp16x2) ||
        !as_pointer(PyTuple_GET_ITEM(centroids_obj, 0), &centroids) ||
        !as_u32(PyTuple_GET_ITEM(centroids_obj, 1), &clusters))
      return nullptr;
    if (PyTuple_Check(assignments_obj)) {
      if (PyTuple_GET_SIZE(assignments_obj) != 2) {
        PyErr_SetString(PyExc_ValueError, "\"assignments\" must be a pointer or a tuple of length 2");
        return nullptr;
      }
      if (!as_pointer(PyTuple_GET_ITEM(assignments_obj, 0), &assignments) ||
          !as_pointer(PyTuple_GET_ITEM(assignments_obj, 1), &neighbors))
        return nullptr;
    } else if (!as_pointer(assignments_obj, &assignments)) {
      return nullptr;
    }
    if (!samples || !centroids || !assignments) {
      PyErr_SetString(PyExc_ValueError, "null pointer");
      return nullptr;
    }
  } else {
    if (!take_samples(samples_obj, &keep_s, &samples, &fp16x2, &n, &d)) return nullptr;
    keep_c.reset(PyArray_FROM_OTF(centroids_obj, fp16x2 ? NPY_FLOAT16 : NPY_FLOAT32, NPY_ARRAY_IN_ARRAY));
    if (!keep_c.p) {
      PyErr_Clear();
      PyErr_SetString(PyExc_TypeError, "\"centroids\" must be a 2D float32 or float16 numpy array");
      return nullptr;
    }
    if (PyArray_NDIM(keep_c.arr()) != 2) {
      PyErr_SetString(PyExc_ValueError, "\"centroids\" must be a 2D numpy array");
      return nullptr;
    }
    clusters = static_cast<uint32_t>(PyArray_DIM(keep_c.arr(), 0));
    if (static_cast<uint32_t>(PyArray_DIM(keep_c.arr(), 1)) != (fp16x2 ? d * 2 : d)) {
      PyErr_SetString(PyExc_ValueError, "\"centroids\" must have same number of features as \"samples\"");
      return nullptr;
    }
    centroids = static_cast<float*>(PyArray_DATA(keep_c.arr()));
    keep_a.reset(PyArray_FROM_OTF(assignments_obj, NPY_UINT32, NPY_ARRAY_IN_ARRAY));
    if (!keep_a.p) {
      PyErr_Clear();
      PyErr_SetString(PyExc_TypeError, "\"assignments\" must be a 1D uint32 numpy array");
      return nullptr;
    }
    if (PyArray_NDIM(keep_a.arr()) != 1) {
      PyErr_SetString(PyExc_ValueError, "\"assignments\" must be a 1D numpy array");
      return nullptr;
    }
    if (static_cast<uint32_t>(PyArray_DIM(keep_a.arr(), 0)) != n) {
      PyErr_SetString(PyExc_ValueError, "\"assignments\" must be of the same length as \"samples\"");
      return nullptr;
    }
    assignments = static_cast<uint32_t*>(PyArray_DATA(keep_a.arr()));
  }
  if (!check_features(d)) return nullptr;
  if (device_ptrs < 0) {
    npy_intp dims[2] = {static_cast<npy_intp>(n), static_cast<npy_intp>(k)};
    neighbors_arr.reset(PyArray_EMPTY(2, dims, NPY_UINT32, 0));
    if (!neighbors_arr.p) return nullptr;
    neighbors = static_cast<uint32_t*>(PyArray_DATA(neighbors_arr.arr()));
  } else if (!neighbors) {
    void* nb = nullptr;
    int rc = kmcuda_b200_device_malloc(device_ptrs, static_cast<uint64_t>(n) * k * 4, &nb);
    if (rc != kmcudaSuccess) return raise_for(rc, "knn_cuda");
    neighbors = static_cast<uint32_t*>(nb);
  }
  int result;
  Py_BEGIN_ALLOW_THREADS
  result = knn_cuda(static_cast<uint16_t>(k), metric, n, static_cast<uint16_t>(d), clusters, device, device_ptrs, fp16x2,
                    verbosity, samples, centroids, assignments, neighbors);
  Py_END_ALLOW_THREADS
  if (result != kmcudaSuccess) return raise_for(result, "knn_cuda");
  if (device_ptrs < 0) return Py_BuildValue("O", neighbors_arr.p);
  return Py_BuildValue("K", static_cast<unsigned long long>(reinterpret_cast<uintptr_t>(neighbors)));
}

char module_doc[] = "K-means and K-nn on NVIDIA H100 (drop-in for src-d/kmcuda's libKMCUDA).";
char kmeans_doc[] = "kmeans_cuda(samples, clusters, tolerance=.01, init=\"k-means++\", yinyang_t=.1, metric=\"L2\", "
                    "average_distance=False, seed=time(), device=0, verbosity=0, sample_weight=None, batch_size=None, "
                    "max_steps=0, relocate_empty_clusters=False, n_init=1, inertia=False, bisecting=None, max_iter=0, "
                    "tol=None, n_iter=False, init_size=None) -> (centroids, assignments[, avg][, inertia][, n_iter]).  The keywords "
                    "are described in the kmcuda_b200 package's docstring.";
char knn_doc[] = "knn_cuda(k, samples, centroids, assignments, metric=\"L2\", device=0, verbosity=0) -> neighbors";

PyMethodDef module_functions[] = {
    {"kmeans_cuda", reinterpret_cast<PyCFunction>(py_kmeans_cuda), METH_VARARGS | METH_KEYWORDS, kmeans_doc},
    {"knn_cuda", reinterpret_cast<PyCFunction>(py_knn_cuda), METH_VARARGS | METH_KEYWORDS, knn_doc},
    {nullptr, nullptr, 0, nullptr}};

PyModuleDef module_def = {PyModuleDef_HEAD_INIT, "libKMCUDA", module_doc, -1, module_functions,
                          nullptr, nullptr, nullptr, nullptr};

}  // namespace

extern "C" {
PyMODINIT_FUNC PyInit_libKMCUDA(void) {
  PyObject* m = PyModule_Create(&module_def);
  if (!m) return nullptr;
  import_array();
  Py_INCREF(Py_True);
  if (PyModule_AddObject(m, "supports_fp16", Py_True) < 0) {
    Py_DECREF(Py_True);
    Py_DECREF(m);
    return nullptr;
  }
  return m;
}
}
