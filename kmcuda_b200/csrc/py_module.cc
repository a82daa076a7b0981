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

void* as_pointer(PyObject* o) {
  return reinterpret_cast<void*>(static_cast<uintptr_t>(PyLong_AsUnsignedLongLong(o)));
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
    *data = static_cast<const float*>(as_pointer(obj));
    if (PyErr_Occurred()) return false;
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

PyObject* py_kmeans_cuda(PyObject*, PyObject* args, PyObject* kwargs) {
  uint32_t clusters = 0, afkmc2_m = 0, seed = static_cast<uint32_t>(time(nullptr)), device = 0;
  int32_t verbosity = 0;
  int adflag = 0;
  float tolerance = .01f, yinyang_t = .1f;
  PyObject *samples_obj, *init_obj = Py_None, *metric_obj = Py_None, *weight_obj = Py_None;
  static const char* kwlist[] = {"samples", "clusters", "tolerance", "init", "yinyang_t", "metric",
                                 "average_distance", "seed", "device", "verbosity", "sample_weight", nullptr};
  if (!PyArg_ParseTupleAndKeywords(args, kwargs, "OI|fOfOpIIiO", const_cast<char**>(kwlist), &samples_obj,
                                   &clusters, &tolerance, &init_obj, &yinyang_t, &metric_obj, &adflag, &seed,
                                   &device, &verbosity, &weight_obj))
    return nullptr;
  KMCUDAInitMethod init = kmcudaInitMethodPlusPlus;
  auto named_init = [&init](PyObject* o) {
    const char* s = PyUnicode_Check(o) ? PyUnicode_AsUTF8(o) : nullptr;
    if (s && (strcmp(s, "k-means||") == 0 || strcmp(s, "kmeans||") == 0)) {   // kmcuda_b200.h, not in kmcuda.h's table
      init = kmcudaInitMethodKMeansParallel;
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
    if (PyTuple_Size(init_obj) > 1 && init == kmcudaInitMethodAFKMC2)
      afkmc2_m = static_cast<uint32_t>(PyLong_AsUnsignedLong(PyTuple_GetItem(init_obj, 1)));
    if (PyTuple_Size(init_obj) > 1 && init == kmcudaInitMethodKMeansParallel) {   // rounds: an integer in [0, 32]
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
        PyErr_SetString(PyExc_ValueError, "k-means|| rounds must be an integer in [0, 32]");
        return nullptr;
      }
      afkmc2_m = static_cast<uint32_t>(v);
    }
  } else {
    init = kmcudaInitMethodImport;
  }
  KMCUDADistanceMetric metric;
  if (!parse_metric(metric_obj, &metric)) return nullptr;
  if (clusters < 2 || clusters == UINT32_MAX) {
    PyErr_SetString(PyExc_ValueError, "\"clusters\" must be greater than 1 and less than (1 << 32) - 1");
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
    PyObject* ptr = PyTuple_GetItem(samples_obj, 0);
    PyObject* shape = PyTuple_GetItem(samples_obj, 2);
    if (!PyLong_Check(ptr)) {
      PyErr_SetString(PyExc_ValueError, "\"samples\"[0] is not a pointer (integer)");
      return nullptr;
    }
    samples = static_cast<float*>(as_pointer(ptr));
    if (!samples) {
      PyErr_SetString(PyExc_ValueError, "\"samples\"[0] is null");
      return nullptr;
    }
    device_ptrs = static_cast<int>(PyLong_AsLong(PyTuple_GetItem(samples_obj, 1)));
    if (!PyTuple_Check(shape) || (PyTuple_GET_SIZE(shape) != 2 && PyTuple_GET_SIZE(shape) != 3)) {
      PyErr_SetString(PyExc_TypeError, "\"samples\"[2] must be a shape tuple");
      return nullptr;
    }
    n = static_cast<uint32_t>(PyLong_AsUnsignedLong(PyTuple_GetItem(shape, 0)));
    d = static_cast<uint32_t>(PyLong_AsUnsignedLong(PyTuple_GetItem(shape, 1)));
    if (PyTuple_GET_SIZE(shape) == 3) fp16x2 = PyObject_IsTrue(PyTuple_GetItem(shape, 2)) == 1;
    if (size == 5) {
      centroids = static_cast<float*>(as_pointer(PyTuple_GetItem(samples_obj, 3)));
      assignments = static_cast<uint32_t*>(as_pointer(PyTuple_GetItem(samples_obj, 4)));
    }
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
  int result;
  Py_BEGIN_ALLOW_THREADS
  if (weights)
    result = kmcuda_b200_kmeans_weighted(init, &afkmc2_m, tolerance, yinyang_t, metric, n, static_cast<uint16_t>(d),
                                         clusters, seed, device, device_ptrs, fp16x2, verbosity, samples, weights,
                                         centroids, assignments, adflag ? &average_distance : nullptr);
  else
    result = kmeans_cuda(init, &afkmc2_m, tolerance, yinyang_t, metric, n, static_cast<uint16_t>(d), clusters, seed,
                         device, device_ptrs, fp16x2, verbosity, samples, centroids, assignments,
                         adflag ? &average_distance : nullptr);
  Py_END_ALLOW_THREADS
  if (result != kmcudaSuccess) return raise_for(result, "kmeans_cuda");
  if (device_ptrs < 0) {
    if (!adflag) return Py_BuildValue("OO", centroids_arr.p, assignments_arr.p);
    return Py_BuildValue("OOf", centroids_arr.p, assignments_arr.p, average_distance);
  }
  const unsigned long long cp = reinterpret_cast<uintptr_t>(centroids), ap = reinterpret_cast<uintptr_t>(assignments);
  if (!adflag) return Py_BuildValue("KK", cp, ap);
  return Py_BuildValue("KKf", cp, ap, average_distance);
}

PyObject* py_knn_cuda(PyObject*, PyObject* args, PyObject* kwargs) {
  uint32_t device = 0, k = 0;
  int32_t verbosity = 0;
  PyObject *samples_obj, *centroids_obj, *assignments_obj, *metric_obj = Py_None;
  static const char* kwlist[] = {"k", "samples", "centroids", "assignments", "metric", "device", "verbosity", nullptr};
  if (!PyArg_ParseTupleAndKeywords(args, kwargs, "IOOO|OIi", const_cast<char**>(kwlist), &k, &samples_obj,
                                   &centroids_obj, &assignments_obj, &metric_obj, &device, &verbosity))
    return nullptr;
  KMCUDADistanceMetric metric;
  if (!parse_metric(metric_obj, &metric)) return nullptr;
  if (k == 0 || k > UINT16_MAX) {
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
    samples = static_cast<float*>(as_pointer(PyTuple_GetItem(samples_obj, 0)));
    device_ptrs = static_cast<int>(PyLong_AsLong(PyTuple_GetItem(samples_obj, 1)));
    PyObject* shape = PyTuple_GetItem(samples_obj, 2);
    if (!PyTuple_Check(shape) || (PyTuple_GET_SIZE(shape) != 2 && PyTuple_GET_SIZE(shape) != 3)) {
      PyErr_SetString(PyExc_TypeError, "\"samples\"[2] must be a shape tuple");
      return nullptr;
    }
    n = static_cast<uint32_t>(PyLong_AsUnsignedLong(PyTuple_GetItem(shape, 0)));
    d = static_cast<uint32_t>(PyLong_AsUnsignedLong(PyTuple_GetItem(shape, 1)));
    if (PyTuple_GET_SIZE(shape) == 3) fp16x2 = PyObject_IsTrue(PyTuple_GetItem(shape, 2)) == 1;
    centroids = static_cast<float*>(as_pointer(PyTuple_GetItem(centroids_obj, 0)));
    clusters = static_cast<uint32_t>(PyLong_AsUnsignedLong(PyTuple_GetItem(centroids_obj, 1)));
    if (PyTuple_Check(assignments_obj)) {
      if (PyTuple_GET_SIZE(assignments_obj) != 2) {
        PyErr_SetString(PyExc_ValueError, "\"assignments\" must be a pointer or a tuple of length 2");
        return nullptr;
      }
      assignments = static_cast<uint32_t*>(as_pointer(PyTuple_GetItem(assignments_obj, 0)));
      neighbors = static_cast<uint32_t*>(as_pointer(PyTuple_GetItem(assignments_obj, 1)));
    } else {
      assignments = static_cast<uint32_t*>(as_pointer(assignments_obj));
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
                    "average_distance=False, seed=time(), device=0, verbosity=0, sample_weight=None) -> "
                    "(centroids, assignments[, avg])";
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
