// _hostcall: the Python-facing call of the flagship's per-step entry, agx_hp1_position_task_step_at, without ctypes.
//
// The device takes ~9 us per chained step; a ctypes call alone costs ~1 us of the host's enqueue (argument conversion objects per
// call), a METH_FASTCALL function a tenth of that.  Hp1Engine hands over the entry's address in the loaded library, so the library
// named by AGX_LIB_PATH is the one called.
#define PY_SSIZE_T_CLEAN
#include <Python.h>
#include <stdint.h>

namespace {

using StepAt = int (*)(const void* cfg, const void* buf, void* stream, uint32_t step_index);

// step_at(entry, cfg, buf, stream, step_index) -> int: entry(cfg, buf, stream, step_index), every argument an int (an address; stream
// may be 0 = the legacy default stream)
PyObject* step_at(PyObject*, PyObject* const* args, Py_ssize_t nargs) {
    if (nargs != 5) {
        PyErr_SetString(PyExc_TypeError, "step_at(entry, cfg, buf, stream, step_index) takes 5 integer arguments");
        return nullptr;
    }
    void* p[4];
    for (int i = 0; i < 4; ++i) {
        p[i] = PyLong_AsVoidPtr(args[i]);
        if (!p[i] && PyErr_Occurred()) return nullptr;
    }
    const unsigned long t = PyLong_AsUnsignedLong(args[4]);
    if (t == (unsigned long)-1 && PyErr_Occurred()) return nullptr;
    if (!p[0] || t > 0xffffffffUL) {
        PyErr_SetString(PyExc_ValueError, "step_at: NULL entry or step_index above 32 bits");
        return nullptr;
    }
    return PyLong_FromLong(reinterpret_cast<StepAt>(p[0])(p[1], p[2], p[3], (uint32_t)t));
}

PyMethodDef methods[] = {
    {"step_at", reinterpret_cast<PyCFunction>(reinterpret_cast<void (*)(void)>(step_at)), METH_FASTCALL,
     "step_at(entry, cfg, buf, stream, step_index) -> int"},
    {nullptr, nullptr, 0, nullptr},
};
PyModuleDef module = {PyModuleDef_HEAD_INIT, "_hostcall", nullptr, -1, methods};

}  // namespace

PyMODINIT_FUNC PyInit__hostcall(void) { return PyModule_Create(&module); }
