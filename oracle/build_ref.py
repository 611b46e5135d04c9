"""Recipe: the reference's own `prune` (partition/ply_c/ply_c.cpp:149-380) as a plain shared library, for comparison.

    SPG_REFERENCE=<superpoint_graph checkout> python oracle/build_ref.py

The reference builds ply_c against Boost.Python and Eigen, but `class AttributeGrid` and `prune` use neither in any
real way: a std::map keyed on a boost::tuple of three uint32 (whose comparison is the lexicographic `<` of a
std::tuple), `bp::len` and `ndarray::get_data`.  This recipe cuts exactly that text out of the checkout between two
markers, checks it against a recorded sha256 (a different revision fails loudly), and compiles it with the
reference's flags (g++ -std=c++11 -fopenmp -O3) after a prelude that supplies those few names and a C entry point.
Nothing of the reference is stored in this repository: the extract lives only in the build directory and the
library lands in oracle/_ref/ (git-ignored).

load_prune() returns a ctypes-backed prune(xyz, voxel_size, rgb, labels, objects, n_labels, n_objects) with the
reference's semantics (uint8 labels and uint32 objects, as its pointers read them), or None if the library was
not built.
"""
import ctypes
import hashlib
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT_DIR, "libply_c_prune.so")
SOURCE = os.path.join("partition", "ply_c", "ply_c.cpp")
START = "class AttributeGrid {"
END = "    return to_py_tuple::convert(Custom_tuple(pruned_xyz,pruned_rgb, pruned_labels, pruned_objects));\n}"
SHA256 = "bc6c4440e2e1be5b627e54fcf39cf28c8f1f0bc83ccf78078667bbbac9c0bba2"
FLAGS = ["-std=c++11", "-fopenmp", "-O3", "-fPIC", "-shared"]

PRELUDE = r"""
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <iterator>
#include <limits>
#include <map>
#include <sstream>
#include <stdexcept>
#include <tuple>
#include <vector>

struct PyObject;
namespace shim {
struct ndarray {
    char* data;
    uint64_t rows;
    char* get_data() const { return data; }
};
inline uint64_t len(const ndarray& a) { return a.rows; }
}  // namespace shim
namespace bp = shim;
namespace bpn = shim;

typedef std::tuple<uint32_t, uint32_t, uint32_t> Space_tuple;

struct Custom_tuple {
    std::vector<std::vector<float> > xyz;
    std::vector<std::vector<uint8_t> > rgb;
    std::vector<std::vector<uint32_t> > labels, objects;
    Custom_tuple(const std::vector<std::vector<float> >& a, const std::vector<std::vector<uint8_t> >& b,
                 const std::vector<std::vector<uint32_t> >& c, const std::vector<std::vector<uint32_t> >& d)
        : xyz(a), rgb(b), labels(c), objects(d) {}
};

static Custom_tuple* g_result = nullptr;

struct to_py_tuple {
    static PyObject* convert(const Custom_tuple& t) {
        delete g_result;
        g_result = new Custom_tuple(t);
        return nullptr;
    }
};
"""

ENTRY = r"""
extern "C" {

// 0: ok, result kept for ref_prune_fetch; 1: std::out_of_range (the reference's IndexError); 2: another exception
int ref_prune(const float* xyz, int64_t n, float voxel_size, const uint8_t* rgb, const uint8_t* labels,
              const uint32_t* objects, int n_labels, int n_objects, int64_t* shape) {
    shim::ndarray a_xyz = {(char*)xyz, (uint64_t)n}, a_rgb = {(char*)rgb, (uint64_t)n};
    shim::ndarray a_lab = {(char*)labels, (uint64_t)n}, a_obj = {(char*)objects, (uint64_t)n};
    std::ostringstream sink;
    std::streambuf* saved = std::cout.rdbuf(sink.rdbuf());  // prune's progress lines
    int rc = 0;
    try {
        prune(a_xyz, voxel_size, a_rgb, a_lab, a_obj, n_labels, n_objects);
    } catch (const std::out_of_range&) {
        rc = 1;
    } catch (...) {
        rc = 2;
    }
    std::cout.rdbuf(saved);
    if (rc) return rc;
    shape[0] = (int64_t)g_result->xyz.size();
    shape[1] = (int64_t)g_result->labels[0].size();   // VecvecToArray's column count: row 0
    shape[2] = (int64_t)g_result->objects[0].size();
    return 0;
}

void ref_prune_fetch(float* xyz, uint8_t* rgb, uint32_t* labels, uint32_t* objects) {
    const size_t m = g_result->xyz.size(), cl = g_result->labels[0].size(), co = g_result->objects[0].size();
    for (size_t i = 0; i < m; ++i) {
        std::memcpy(xyz + 3 * i, g_result->xyz[i].data(), 3 * sizeof(float));
        std::memcpy(rgb + 3 * i, g_result->rgb[i].data(), 3);
        std::memcpy(labels + cl * i, g_result->labels[i].data(), cl * sizeof(uint32_t));
        std::memcpy(objects + co * i, g_result->objects[i].data(), co * sizeof(uint32_t));
    }
}

}  // extern "C"
"""


def extract(reference):
    """The text of `class AttributeGrid` ... the end of `prune`, checked against the recorded sha256."""
    text = open(os.path.join(reference, SOURCE)).read()
    a = text.find(START)
    b = text.find(END, a) if a >= 0 else -1
    if a < 0 or b < 0:
        raise RuntimeError("%s: the prune markers are not there; not the expected reference revision" % SOURCE)
    body = text[a:b + len(END)] + "\n"
    digest = hashlib.sha256(body.encode()).hexdigest()
    if digest != SHA256:
        raise RuntimeError("%s: the prune extract has sha256 %s, expected %s; not the expected reference revision"
                           % (SOURCE, digest, SHA256))
    return body


def build(reference, out=LIB, verbose=True):
    cxx = shutil.which("g++") or shutil.which("c++")
    if not cxx:
        raise RuntimeError("no C++ compiler found to build the reference prune")
    body = extract(reference)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "ply_c_prune.cpp")
        with open(src, "w") as f:
            f.write(PRELUDE + "\n" + body + "\n" + ENTRY)
        cmd = [cxx] + FLAGS + [src, "-o", out]
        if verbose:
            print("[ref build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return out


def load_prune(path=LIB):
    """ctypes prune with the reference's semantics, or None when the library was not built."""
    if not os.path.exists(path):
        return None
    import numpy as np

    dll = ctypes.CDLL(path)
    dll.ref_prune.restype = ctypes.c_int
    dll.ref_prune.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                              ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    dll.ref_prune_fetch.restype = None
    dll.ref_prune_fetch.argtypes = [ctypes.c_void_p] * 4

    def prune(xyz, voxel_size, rgb, labels, objects, n_labels, n_objects):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32)
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        lab = np.ascontiguousarray(labels, dtype=np.uint8) if n_labels > 0 else np.zeros(1, np.uint8)
        obj = np.ascontiguousarray(objects, dtype=np.uint32) if n_objects > 0 else np.zeros(1, np.uint32)
        shape = np.zeros(3, np.int64)
        rc = dll.ref_prune(xyz.ctypes.data, xyz.shape[0], float(voxel_size), rgb.ctypes.data, lab.ctypes.data,
                           obj.ctypes.data, int(n_labels), int(n_objects), shape.ctypes.data)
        if rc == 1:
            raise IndexError("vector::_M_range_check")
        if rc:
            raise RuntimeError("the reference prune raised")
        m, cl, co = (int(v) for v in shape)
        out = (np.empty((m, 3), np.float32), np.empty((m, 3), np.uint8), np.empty((m, cl), np.uint32),
               np.empty((m, co), np.uint32))
        dll.ref_prune_fetch(*(a.ctypes.data for a in out))
        return out

    return prune


if __name__ == "__main__":
    ref = os.environ.get("SPG_REFERENCE")
    if not ref:
        sys.exit("set SPG_REFERENCE to a superpoint_graph checkout")
    print(build(ref))
