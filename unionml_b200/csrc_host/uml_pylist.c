/* CPython glue for the predictor contract `-> List[float]` (unionml:README.md:87-92).
 *
 * The canonical predictor returns `[float(x) for x in estimator.predict(features)]`: one Python float per row.
 * Creating 10M float objects costs ~0.25 s on the GPU box's host - more than the whole H2D + GPU pipeline (0.12 s).
 * Labels take only n_classes distinct values, so the list can reference n_classes float objects instead of allocating
 * one per row (floats are immutable; equality, type and repr are those of `float(x)`): filling list slots from an
 * int32 label vector is a pointer store and a reference-count increment per row, ~2 ns.
 *
 * Loaded with ctypes.PyDLL (the GIL stays held); not part of the CUDA library's C ABI (include/uml_b200.h).
 */
#define PY_SSIZE_T_CLEAN
#include <Python.h>
#include <stdint.h>

/* list[start + i] = table[labels[i]] for i in [0, count); list is a pre-sized list, table a list of floats.
 * Returns 0, or -1 with a Python exception set. */
int uml_list_fill_from_labels(PyObject* list, Py_ssize_t start, const int32_t* labels, Py_ssize_t count, PyObject* table) {
  if (!PyList_CheckExact(list) || !PyList_CheckExact(table)) {
    PyErr_SetString(PyExc_TypeError, "uml_list_fill_from_labels: list and table must be lists");
    return -1;
  }
  const Py_ssize_t n = PyList_GET_SIZE(list), n_classes = PyList_GET_SIZE(table);
  if (start < 0 || count < 0 || start + count > n) {
    PyErr_SetString(PyExc_IndexError, "uml_list_fill_from_labels: range outside the list");
    return -1;
  }
  for (Py_ssize_t i = 0; i < count; ++i) {
    const int32_t k = labels[i];
    if (k < 0 || k >= n_classes) {
      PyErr_Format(PyExc_ValueError, "label %d at row %zd outside [0, %zd)", (int)k, start + i, n_classes);
      return -1;
    }
    PyObject* item = PyList_GET_ITEM(table, k);
    PyObject* old = PyList_GET_ITEM(list, start + i);
    Py_INCREF(item);
    PyList_SET_ITEM(list, start + i, item);
    Py_XDECREF(old);
  }
  return 0;
}
