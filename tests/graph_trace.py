"""Call traces of the host-side graph (neuronika_b200/csrc/nk_graph.cpp) over a recording stub of the kernel ABI.

nk_graph.cpp is host code whose only effect on the device is the sequence of nk_* calls it makes.  This module
generates a stub of every function declared in include/nk_b200.h that records each call (name and arguments) as one
line of text, compiles it together with nk_graph.cpp into a shared library with the host C++ compiler, and drives the
graph through the nkg_* prototypes of neuronika_b200/variable.py over a corpus of scenarios.  Two builds of the graph
that produce the same traces launch the same device work.

How arguments are written:
  - device pointers as allocation ordinal plus byte offset: `d7` (nk_alloc / nk_alloc_uninit), `x3` (memory the
    scenario owns: caller-owned gradients, external leaves, optimizer state, reduce-scatter slots), `d7+4096`;
    NULL as `0`;
  - host arrays (shapes, lens, operand tables) by content, with the length taken from the call's count argument;
  - floats with 9 significant digits; the context (always the same) is left out.
Hooks write into the same trace, so their timing relative to the launches is part of it, and so are the
nkg_last_error() texts of the error scenarios.  `stub_fail(name)` makes a function return NK_ERR_UNSUPPORTED.

tests/golden/make_graph_trace.py writes tests/golden/graph_trace.json; tests/test_graph_trace.py compares."""
from __future__ import annotations

import ctypes as C
import gc
import os
import re
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nk_b200.h")
GRAPH_SRC = os.path.join(ROOT, "neuronika_b200", "csrc", "nk_graph.cpp")
GOLDEN = os.path.join(ROOT, "tests", "golden", "graph_trace.json")

F32, BF16 = 0, 1
NK_ERR_UNSUPPORTED = -5

# host arrays among the ABI's pointer parameters: (function, parameter) -> parameter holding the element count
HOST_ARRAYS = {
    ("nk_add_bcast_fwd", "y_shape"): "y_ndim", ("nk_add_bcast_fwd", "l_shape"): "l_ndim",
    ("nk_add_bcast_fwd", "r_shape"): "r_ndim",
    ("nk_unbroadcast_acc", "dst_shape"): "dst_ndim", ("nk_unbroadcast_acc", "g_shape"): "g_ndim",
    ("nk_binary_bcast_fwd", "y_shape"): "y_ndim", ("nk_binary_bcast_fwd", "l_shape"): "l_ndim",
    ("nk_binary_bcast_fwd", "r_shape"): "r_ndim",
    ("nk_binary_bcast_bwd", "l_shape"): "l_ndim", ("nk_binary_bcast_bwd", "r_shape"): "r_ndim",
    ("nk_transpose", "src_shape"): "ndim",
    ("nk_padnd_fwd", "in_sp"): "nsp", ("nk_padnd_fwd", "pad"): "nsp",
    ("nk_padnd_bwd", "in_sp"): "nsp", ("nk_padnd_bwd", "pad"): "nsp",
    **{(f, p): "nsp" for f in ("nk_convnd_fwd", "nk_convnd_bwd_input", "nk_convnd_bwd_kernel")
       for p in ("in_sp", "k", "stride", "dilation")},
    ("nk_chunk_fwd", "x_shape"): "ndim", ("nk_chunk_fwd", "chunk_shape"): "ndim",
    ("nk_chunk_bwd", "x_shape"): "ndim", ("nk_chunk_bwd", "chunk_shape"): "ndim",
    ("nk_cat_fwd", "xs"): "count", ("nk_cat_fwd", "lens"): "count",
    ("nk_cat_bwd", "dxs"): "count", ("nk_cat_bwd", "dx_dtypes"): "count", ("nk_cat_bwd", "betas"): "count",
    ("nk_cat_bwd", "lens"): "count",
    ("nk_gemm_rs", "slots"): "world",
    **{(f, p): "count" for f in ("nk_multi_sgd_step", "nk_multi_adam_step", "nk_multi_rmsprop_step",
                                 "nk_multi_adagrad_step")
       for p in ("w", "g", "n", "master", "momentum_buf", "exp_avg", "exp_avg_sq", "max_exp_avg_sq", "square_avg",
                 "grad_avg", "grad_sq")},
}


def header_functions():
    """[(return type, name, [(type, name), ...])] of every nk_* function declared in include/nk_b200.h"""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    out = []
    for m in re.finditer(r"([A-Za-z_][\w\s]*?\**)\s*\b(nk_[a-z0-9_]+)\s*\(([^;{}()]*)\)\s*;", text):
        ret = " ".join(m.group(1).split()[-2:]) if m.group(1).split()[-2:-1] == ["const"] else m.group(1).split()[-1]
        params = []
        for p in m.group(3).split(","):
            p = " ".join(p.split())
            if p in ("", "void"):
                continue
            pm = re.match(r"(.*?)\s*\b(\w+)$", p)
            params.append((re.sub(r"\s*\*", "*", pm.group(1)).strip(), pm.group(2)))
        out.append((ret, m.group(2), params))
    return out


_RUNTIME = r"""
#include <stdint.h>
#include <stdio.h>
#include <set>
#include <string>
#include <vector>
#include "nk_b200.h"

namespace {
std::string g_trace, g_taken, g_fmt;
std::set<std::string> g_fail;
struct Range { uintptr_t base; size_t bytes; std::string label; };
std::vector<Range> g_ranges;
uintptr_t g_next = 0x100000000ull;
int g_dev = 0, g_ext = 0;

uintptr_t new_range(size_t bytes, const std::string& label) {
  const uintptr_t base = g_next;
  g_next += (bytes + 255) / 256 * 256 + 65536;
  g_ranges.push_back({base, bytes, label});
  return base;
}
std::string tr_ptr(const void* p) {
  if (!p) return "0";
  const uintptr_t a = (uintptr_t)p;
  for (const Range& r : g_ranges)
    if (a >= r.base && a <= r.base + r.bytes)
      return a == r.base ? r.label : r.label + "+" + std::to_string(a - r.base);
  char b[32];
  snprintf(b, sizeof b, "?%llx", (unsigned long long)a);
  return b;
}
std::string tr_int(long long v) { return std::to_string(v); }
std::string tr_flt(double v) {
  char b[32];
  snprintf(b, sizeof b, "%.9g", v);
  return b;
}
template <typename T, typename E>
std::string tr_arr(const T* a, long long n, E each) {
  if (!a) return "0";
  std::string s = "[";
  for (long long i = 0; i < n; ++i) s += (i ? "," : "") + each(a[i]);
  return s + "]";
}
std::string tr_arr(const int64_t* a, long long n) { return tr_arr(a, n, [](int64_t v) { return tr_int(v); }); }
std::string tr_arr(const int* a, long long n) { return tr_arr(a, n, [](int v) { return tr_int(v); }); }
std::string tr_arr(const float* a, long long n) { return tr_arr(a, n, [](float v) { return tr_flt(v); }); }
std::string tr_arr(const void* const* a, long long n) { return tr_arr(a, n, [](const void* v) { return tr_ptr(v); }); }
int rec(const char* name, const std::string& args) {
  g_trace += std::string(name) + "(" + args + ")\n";
  return g_fail.count(name) ? NK_ERR_UNSUPPORTED : NK_OK;
}
}  // namespace

extern "C" {
void stub_reset() {
  g_trace.clear();
  g_fail.clear();
  g_ranges.clear();
  g_dev = g_ext = 0;
}
const char* stub_take() {
  g_taken.swap(g_trace);
  g_trace.clear();
  return g_taken.c_str();
}
void stub_note(const char* line) { g_trace += std::string(line) + "\n"; }
void stub_fail(const char* name) {
  if (name)
    g_fail.insert(name);
  else
    g_fail.clear();
}
void* stub_ext(size_t bytes) { return (void*)new_range(bytes, "x" + std::to_string(g_ext++)); }
const char* stub_fmt(const void* p) {
  g_fmt = tr_ptr(p);
  return g_fmt.c_str();
}

static int alloc(const char* name, size_t bytes, void** dptr) {
  *dptr = (void*)new_range(bytes, "d" + std::to_string(g_dev++));
  g_trace += std::string(name) + "(" + tr_int(bytes) + ") = " + tr_ptr(*dptr) + "\n";
  return NK_OK;
}
int nk_alloc(nk_ctx*, size_t bytes, void** dptr) { return alloc("nk_alloc", bytes, dptr); }
int nk_alloc_uninit(nk_ctx*, size_t bytes, void** dptr) { return alloc("nk_alloc_uninit", bytes, dptr); }
const char* nk_last_error(nk_ctx*) {
  rec("nk_last_error", "");
  return "stub: failure injected by the trace";
}
"""


def _formatter(fn, ptype, pname):
    """C++ expression writing one argument as a std::string"""
    count = HOST_ARRAYS.get((fn, pname))
    if count is not None:
        return "tr_arr(%s, %s)" % (pname, count)
    if ptype == "nk_ctx*":
        return None   # always the graph's context
    if "**" in ptype:
        return 'std::string("out")'
    if "*" in ptype:
        return "tr_ptr(%s)" % pname
    if ptype in ("float", "double"):
        return "tr_flt(%s)" % pname
    return "tr_int((long long)%s)" % pname


def stub_source():
    """C++ source of the recording stub (every nk_* function of the header)"""
    src = [_RUNTIME]
    done = {"nk_alloc", "nk_alloc_uninit", "nk_last_error"}
    for ret, name, params in header_functions():
        if name in done:
            continue
        done.add(name)
        decl = ", ".join("%s %s" % (t, n) for t, n in params)
        fmts = [f for f in (_formatter(name, t, n) for t, n in params) if f]
        args = ' + ", " + '.join(fmts) or 'std::string()'
        body = 'const int rc = rec("%s", %s);' % (name, args)
        if ret == "int":
            tail = "return rc;"
        elif ret.endswith("*"):
            tail = "(void)rc; return %s;" % ('"stub"' if "char" in ret else "nullptr")
        else:
            tail = "(void)rc; return 0;"
        src.append("%s %s(%s) {\n  %s\n  %s\n}" % (ret, name, decl, body, tail))
    src.append("}  // extern \"C\"\n")
    return "\n".join(src)


def compiler():
    for cxx in (os.environ.get("CXX"), "g++", "c++", "clang++"):
        if cxx and shutil.which(cxx):
            return shutil.which(cxx)
    return None


def build_library(workdir, graph_src=GRAPH_SRC):
    """compile the stub and nk_graph.cpp into workdir/libnkg_trace.so; returns its path"""
    stub = os.path.join(workdir, "nk_stub.cpp")
    with open(stub, "w") as fh:
        fh.write(stub_source())
    out = os.path.join(workdir, "libnkg_trace.so")
    cmd = [compiler(), "-std=c++17", "-O1", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"), stub, graph_src,
           "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building the traced graph failed:\n" + r.stderr[-4000:])
    return out


# ------------------------------------------------------------------------------------------------------------- driver
class NkgError(Exception):
    pass


class Graph:
    """the nkg_* surface bound to the stub library, with handles that are released like the Python temporaries of
    neuronika_b200.variable (fusion decisions depend on which tensors are still held)"""

    def __init__(self, path):
        from neuronika_b200.variable import _G
        self.lib = C.CDLL(path)
        for name, (restype, argtypes) in _G.items():
            f = getattr(self.lib, name)
            f.restype, f.argtypes = restype, argtypes
        self.lib.stub_take.restype = C.c_char_p
        self.lib.stub_note.argtypes = [C.c_char_p]
        self.lib.stub_fail.argtypes = [C.c_char_p]
        self.lib.stub_ext.restype = C.c_void_p
        self.lib.stub_ext.argtypes = [C.c_size_t]
        self.lib.stub_fmt.restype = C.c_char_p
        self.lib.stub_fmt.argtypes = [C.c_void_p]
        self.ctx = C.c_void_p(0x1000)
        self.other_ctx = C.c_void_p(0x2000)
        self._keep = []

    # ---- trace control
    def run(self, scenario):
        """the trace of one scenario.  Handles are released by reference counting, as in neuronika_b200.variable; the
        cycle collector is held off so that it cannot release one at a random point.  The frees of the teardown (the
        scenario's handles going out of scope, in whatever order Python clears them) end the trace as one line: how
        many there were and which device allocations were never freed."""
        self.lib.stub_reset()
        self.lib.nkg_set_fusion(1)
        gc.disable()
        try:
            scenario(self)
            self._keep = []
            gc.collect(0)
        finally:
            gc.enable()
            self.lib.nkg_set_fusion(1)
        lines = self.lib.stub_take().decode().splitlines()
        body = len(lines)
        while body and lines[body - 1].startswith("nk_free("):
            body -= 1
        allocated = {l.rsplit(" = ", 1)[1] for l in lines if l.startswith("nk_alloc")}
        freed = {l[len("nk_free("):-1] for l in lines if l.startswith("nk_free(")}
        return lines[:body] + ["teardown: %d frees, never freed: %s" % (len(lines) - body, sorted(allocated - freed))]

    def note(self, text):
        self.lib.stub_note(str(text).encode())

    def fail(self, name):
        self.lib.stub_fail(name.encode())

    def ext(self, nbytes):
        return self.lib.stub_ext(nbytes)

    def fmt(self, ptr):
        return self.lib.stub_fmt(ptr).decode()

    def fusion(self, level):
        self.lib.nkg_set_fusion(level)

    def ck(self, rc):
        if rc != 0:
            raise NkgError("%d %s" % (rc, self.lib.nkg_last_error().decode()))

    def expect_error(self, fn, *args):
        """run an op that must fail and put its status and message into the trace"""
        try:
            fn(*args)
        except NkgError as e:
            self.note("error " + str(e))
            return
        raise AssertionError("expected an error")

    # ---- handles
    def wrap(self, h):
        return Var(self, h)

    def call(self, name, *args):
        out = C.c_void_p()
        self.ck(getattr(self.lib, name)(*args, C.byref(out)))
        return self.wrap(out)

    def leaf(self, shape, dtype=F32, ctx=None):
        s = (C.c_int64 * max(1, len(shape)))(*shape)
        return self.call("nkg_leaf", ctx or self.ctx, len(shape), s, dtype)

    def param(self, shape, dtype=F32, grad_dtype=None):
        """from_ndarray(...).requires_grad(grad_dtype): the leaf Var is a temporary"""
        return self.leaf(shape, dtype).requires_grad(grad_dtype)

    def external(self, shape, dtype=F32):
        n = 1
        for d in shape:
            n *= d
        s = (C.c_int64 * max(1, len(shape)))(*shape)
        return self.call("nkg_leaf_external", self.ctx, len(shape), s, dtype, C.c_void_p(self.ext(n * 4)))

    def join(self, name, vars, axis):
        hs = (C.c_void_p * len(vars))(*[v.h.value for v in vars])
        out = C.c_void_p()
        self.ck(getattr(self.lib, name)(hs, len(vars), axis, C.byref(out)))
        return self.wrap(out)

    def lstm(self, x, c, h, w_ih, w_hh, b_ih, b_hh):
        oc, oh = C.c_void_p(), C.c_void_p()
        self.ck(self.lib.nkg_lstm_cell(*(v.h if v else None for v in (x, c, h, w_ih, w_hh, b_ih, b_hh)),
                                       C.byref(oc), C.byref(oh)))
        return self.wrap(oc), self.wrap(oh)

    def gru(self, x, h, w_ih, w_hh, b_ih, b_hh):
        oh = C.c_void_p()
        self.ck(self.lib.nkg_gru_cell(*(v.h if v else None for v in (x, h, w_ih, w_hh, b_ih, b_hh)), C.byref(oh)))
        return self.wrap(oh)


_HOOK = C.CFUNCTYPE(None, C.c_void_p, C.c_int64, C.c_int64)
_RS_HOOK = C.CFUNCTYPE(None, C.c_void_p, C.c_int)


def _i64s(vals):
    return (C.c_int64 * max(1, len(vals)))(*vals)


class Var:
    def __init__(self, g, h):
        self.g, self.h = g, h if isinstance(h, C.c_void_p) else C.c_void_p(h)

    def __del__(self):
        if self.h:
            self.g.lib.nkg_release(self.h)
            self.h = None

    def _op(self, name, *args):
        return self.g.call(name, self.h, *args)

    def _bin(self, name, other, *args):
        return self.g.call(name, self.h, other.h if other is not None else None, *args)

    # ---- introspection (written into the trace)
    def describe(self, label):
        lib = self.g.lib
        n = lib.nkg_ndim(self.h)
        s = (C.c_int64 * max(1, n))()
        self.g.ck(lib.nkg_shape(self.h, s))
        self.g.note("%s: diff=%d shape=%s dtype=%d grad_dtype=%d history=%d backward_history=%d" % (
            label, lib.nkg_is_diff(self.h), list(s)[:n], lib.nkg_dtype(self.h), lib.nkg_grad_dtype(self.h),
            lib.nkg_history_len(self.h), lib.nkg_backward_history_len(self.h)))

    def data_ptr(self, label="data"):
        self.g.note("%s -> %s" % (label, self.g.fmt(self.g.lib.nkg_data_ptr(self.h))))

    def grad_ptr(self, label="grad"):
        p = self.g.lib.nkg_grad_ptr(self.h)
        self.g.note("%s -> %s%s" % (label, self.g.fmt(p), "" if p else " (%s)" % self.g.lib.nkg_last_error().decode()))

    # ---- graph
    def requires_grad(self, grad_dtype=None, grad_ptr=None):
        return self.g.call("nkg_requires_grad", self.h, -1 if grad_dtype is None else grad_dtype, grad_ptr)

    def clone(self): return self._op("nkg_clone")
    def forward(self): self.g.ck(self.g.lib.nkg_forward(self.h))
    def backward(self, seed=1.0): self.g.ck(self.g.lib.nkg_backward(self.h, seed))
    def zero_grad(self): self.g.ck(self.g.lib.nkg_zero_grad(self.h))
    def no_grad(self): self.g.ck(self.g.lib.nkg_no_grad(self.h))
    def with_grad(self): self.g.ck(self.g.lib.nkg_with_grad(self.h))

    def set_hook(self, name, row_chunks=1):
        cb = _HOOK(lambda _u, b, e: self.g.note("hook %s [%d, %d)" % (name, b, e)))
        self.g._keep.append(cb)
        self.g.ck(self.g.lib.nkg_set_grad_hook(self.h, C.cast(cb, C.c_void_p), None, row_chunks))

    def set_rs(self, name, world, rank):
        cb = _RS_HOOK(lambda _u, pushed: self.g.note("rs %s pushed=%d" % (name, pushed)))
        slots = (C.c_void_p * world)(*[self.g.ext(1 << 20) for _ in range(world)])
        self.g._keep += [cb, slots]
        self.g.ck(self.g.lib.nkg_set_grad_rs(self.h, world, rank, slots, C.cast(cb, C.c_void_p), None))

    # ---- operators
    def mm(self, o): return self._bin("nkg_mm", o)
    def mm_t(self, o): return self._bin("nkg_mm_t", o)
    def __add__(self, o): return self._bin("nkg_add", o)
    def __sub__(self, o): return self._bin("nkg_sub", o)
    def __mul__(self, o): return self._bin("nkg_mul", o)
    def __truediv__(self, o): return self._bin("nkg_div", o)
    def __neg__(self): return self._op("nkg_neg")
    def unary(self, op, iparam=0): return self._op("nkg_unary", op, iparam)
    def exp(self): return self._op("nkg_exp")
    def ln(self): return self._op("nkg_ln")
    def sqrt(self): return self._op("nkg_sqrt")
    def sigmoid(self): return self._op("nkg_sigmoid")
    def tanh(self): return self._op("nkg_tanh")
    def softplus(self): return self._op("nkg_softplus")
    def leaky_relu(self): return self._op("nkg_leaky_relu")
    def pow(self, e): return self._op("nkg_pow", e)
    def t(self): return self._op("nkg_transpose")
    def mv(self, o): return self._bin("nkg_mv", o)
    def vm(self, o): return self._bin("nkg_vm", o)
    def vv(self, o): return self._bin("nkg_vv", o)
    def relu(self): return self._op("nkg_relu")
    def softmax(self, axis): return self._op("nkg_softmax", axis)
    def log_softmax(self, axis): return self._op("nkg_log_softmax", axis)
    def sum(self): return self._op("nkg_sum")
    def mean(self): return self._op("nkg_mean")
    def mse_loss(self, t, reduction=0): return self._bin("nkg_mse_loss", t, reduction)
    def nll_loss(self, t, reduction=0): return self._bin("nkg_nll_loss", t, reduction)
    def flatten(self): return self._op("nkg_flatten")
    def unsqueeze(self, axis): return self._op("nkg_unsqueeze", axis)
    def pad(self, ph, pw, value=0.0): return self._op("nkg_pad", ph, pw, value)

    def pad_mode(self, padding, mode, value=0.0):
        return self._op("nkg_pad_mode", len(padding), _i64s(padding), mode, value)

    def conv(self, x, stride=(1, 1), dilation=(1, 1), groups=1):
        return self._bin("nkg_convolution", x, *stride, *dilation, groups)

    def conv_nd(self, x, stride, dilation, groups=1):
        return self._bin("nkg_convolution_nd", x, len(stride), _i64s(stride), _i64s(dilation), groups)

    def chunks(self, shape):
        count = C.c_int(0)
        self.g.ck(self.g.lib.nkg_chunks(self.h, len(shape), _i64s(shape), 0, None, C.byref(count)))
        outs = (C.c_void_p * max(1, count.value))()
        self.g.ck(self.g.lib.nkg_chunks(self.h, len(shape), _i64s(shape), count.value, outs, C.byref(count)))
        return [self.g.wrap(C.c_void_p(outs[i])) for i in range(count.value)]

    def cat(self, others, axis): return self.g.join("nkg_cat", [self, *others], axis)
    def stack(self, others, axis): return self.g.join("nkg_stack", [self, *others], axis)

    # ---- SGD through the multi-tensor entry point (state buffers and the nk_optim_hyper block are scenario-owned
    # memory; lr lives in the block)
    def sgd(self, momentum=0.9, master=False):
        n = self.numel()

        def one(p):
            return (C.c_void_p * 1)(p) if p else None
        buf = self.g.ext(n * 4) if momentum else None
        mst = self.g.ext(n * 4) if master else None
        self.g.ck(self.g.lib.nkg_multi_sgd_step((C.c_void_p * 1)(self.h.value), 1, one(buf), one(mst), self.g.ext(24),
                                                0.01, momentum, 0.0, 1 if momentum else 0, 0.5))

    def numel(self):
        n = self.g.lib.nkg_ndim(self.h)
        s = (C.c_int64 * max(1, n))()
        self.g.ck(self.g.lib.nkg_shape(self.h, s))
        out = 1
        for i in range(n):
            out *= s[i]
        return out


# ------------------------------------------------------------------------------------------------------------- corpus
SCENARIOS = {}


def scenario(name):
    def deco(fn):
        SCENARIOS[name] = fn
        return fn
    return deco


def _operand(g, shape, diff, dtype=F32, grad_dtype=None):
    return g.param(shape, dtype, grad_dtype) if diff else g.leaf(shape, dtype)


def _run(g, out, *operands):
    """forward and (when differentiable) backward of `out`, then the gradient pointers of the operands"""
    out.forward()
    if g.lib.nkg_is_diff(out.h):
        out.backward(1.0)
        for i, v in enumerate(operands):
            if g.lib.nkg_is_diff(v.h):
                v.grad_ptr("grad%d" % i)


MIXES = {"dv": (True, False), "vd": (False, True), "dd": (True, True)}
BINARY = {
    "mm": ((4, 6), (6, 5), lambda a, b: a.mm(b)),
    "mm_t": ((4, 6), (5, 6), lambda a, b: a.mm_t(b)),
    "add": ((4, 5), (5,), lambda a, b: a + b),
    "sub": ((3, 4, 5), (4, 1), lambda a, b: a - b),
    "mul": ((3, 4, 5), (4, 1), lambda a, b: a * b),
    "div": ((4, 1), (3, 4, 5), lambda a, b: a / b),
    "mv": ((4, 6), (6,), lambda a, b: a.mv(b)),
    "vm": ((4,), (4, 6), lambda a, b: a.vm(b)),
    "vv": ((7,), (7,), lambda a, b: a.vv(b)),
    "cat": ((3, 2), (3, 4), lambda a, b: a.cat([b], 1)),
    "stack": ((3, 2), (3, 2), lambda a, b: a.stack([b], 0)),
    "conv2d": ((4, 3, 3, 3), (2, 3, 8, 8), lambda k, x: k.conv(x)),
    "conv2d_grouped": ((4, 1, 3, 3), (2, 2, 9, 9), lambda k, x: k.conv(x, (2, 1), (1, 2), 2)),
    "conv1d": ((4, 3, 3), (2, 3, 10), lambda k, x: k.conv_nd(x, (2,), (1,))),
    "conv3d": ((2, 3, 2, 2, 2), (1, 3, 4, 5, 6), lambda k, x: k.conv_nd(x, (1, 2, 1), (1, 1, 2))),
    "mse_mean": ((4, 5), (4, 5), lambda a, b: a.mse_loss(b, 0)),
    "nll_sum": ((4, 5), (4,), lambda a, b: a.nll_loss(b, 1)),
}


def _binary_scenario(ls, rs, op, ld, rd, dtype):
    def run(g):
        a, b = _operand(g, ls, ld, dtype), _operand(g, rs, rd, dtype)
        _run(g, op(a, b), a, b)
    return run


# each side differentiable alone, and both where the node then takes another path than the two halves in sequence
BOTH_SIDES = ("mm_t", "mv", "cat", "conv2d")
for _name, (_ls, _rs, _op) in BINARY.items():
    for _mix, (_ld, _rd) in MIXES.items():
        if _name.startswith(("mse", "nll")) and _rd:
            continue                                   # a differentiable target is an error (see errors)
        if _mix == "dd" and _name not in BOTH_SIDES:
            continue
        SCENARIOS["binary/%s/%s" % (_name, _mix)] = _binary_scenario(_ls, _rs, _op, _ld, _rd, F32)

UNARY = {
    "relu": ((4, 5), lambda a: a.relu()),
    "softmax": ((3, 4, 5), lambda a: a.softmax(1)),
    "log_softmax": ((3, 4), lambda a: a.log_softmax(0)),
    "sum": ((4, 5), lambda a: a.sum()),
    "mean": ((4, 5), lambda a: a.mean()),
    "neg": ((4, 5), lambda a: -a),
    "exp": ((4, 5), lambda a: a.exp()),
    "ln": ((4, 5), lambda a: a.ln()),
    "sqrt": ((4, 5), lambda a: a.sqrt()),
    "sigmoid": ((4, 5), lambda a: a.sigmoid()),
    "tanh": ((4, 5), lambda a: a.tanh()),
    "softplus": ((4, 5), lambda a: a.softplus()),
    "leaky_relu": ((4, 5), lambda a: a.leaky_relu()),
    "pow": ((4, 5), lambda a: a.pow(3)),
    "t": ((2, 3, 4), lambda a: a.t()),
    "pad": ((2, 3, 4, 5), lambda a: a.pad(1, 2, 0.5)),
    "pad_constant_1d": ((2, 3, 7), lambda a: a.pad_mode((2,), 0, 1.5)),
    "pad_reflective_2d": ((1, 2, 5, 6), lambda a: a.pad_mode((1, 2), 1)),
    "pad_replicative_3d": ((1, 1, 3, 4, 5), lambda a: a.pad_mode((1, 1, 2), 2)),
    "flatten": ((2, 3, 4), lambda a: a.flatten().relu()),
    "unsqueeze": ((3, 4), lambda a: a.unsqueeze(1).exp()),
    "chunks_sum": ((4, 6), lambda a: _chunks_sum(a)),
    "cat_repeated": ((2, 3), lambda a: a.cat([a, a], 1)),
    "stack_repeated": ((2, 3), lambda a: a.stack([a], 2)),
}


def _chunks_sum(a):
    cs = a.chunks((2, 3))
    return (cs[0] + cs[3]).sum()


def _unary_scenario(names, dtype, grad_dtype=None):
    def run(g):
        for name in names:
            g.note(name)
            shape, op = UNARY[name]
            a = _operand(g, shape, True, dtype, grad_dtype)
            _run(g, op(a), a)
    return run


UNARY_FAMILIES = {
    "activations": ("relu", "softmax", "log_softmax", "leaky_relu"),
    "reductions": ("sum", "mean"),
    "elementwise": ("neg", "exp", "ln", "sqrt", "sigmoid", "tanh", "softplus", "pow"),
    "padding": ("pad", "pad_constant_1d", "pad_reflective_2d", "pad_replicative_3d"),
    "shapes": ("t", "flatten", "unsqueeze", "chunks_sum", "cat_repeated", "stack_repeated"),
}
assert sorted(n for f in UNARY_FAMILIES.values() for n in f) == sorted(UNARY)
for _family, _names in UNARY_FAMILIES.items():
    SCENARIOS["unary/%s" % _family] = _unary_scenario(_names, F32)
# an f32 gradient on a bf16 leaf: kernels that produce bf16 write a temporary that is added into the gradient
SCENARIOS["unary/bf16_leaf_f32_grad"] = _unary_scenario(("relu", "softmax", "exp", "pad", "pad_constant_1d", "t"),
                                                        BF16, F32)


@scenario("mixed_dtype_gradients")
def _mixed_dtype_gradients(g):
    k = g.leaf((4, 3, 3, 3), BF16)
    x = g.param((2, 3, 8, 8), BF16, F32)
    _run(g, k.conv(x), x)
    k1 = g.leaf((4, 3, 3), BF16)
    x1 = g.param((2, 3, 10), BF16, F32)
    _run(g, k1.conv_nd(x1, (1,), (2,)), x1)
    kd = g.param((4, 3, 3, 3), BF16, F32)
    xd = g.param((2, 3, 8, 8), BF16, F32)
    _run(g, kd.conv(xd), kd, xd)
    xm = g.param((4, 5), BF16, F32)
    _run(g, xm.mse_loss(g.leaf((4, 5), BF16)), xm)
    xn = g.param((4, 5), BF16, F32)
    _run(g, xn.nll_loss(g.leaf((4,), F32)), xn)
    xs = g.param((3, 4), BF16, F32)
    _run(g, xs.mm(g.leaf((4, 2), BF16)), xs)


# ---- Linear + ReLU MLP (nn.Linear: input.mm_t(weight) + bias)
def _mlp(g, level, steps=1, keep_pre=False, hooks=None, rs=None, zero=True, fail=None, sizes=(256, 256, 16)):
    g.fusion(level)
    if fail:
        g.fail(fail)
    n = 64
    x = g.leaf((n, sizes[0]), BF16)
    target = g.leaf((n, sizes[-1]), BF16)
    layers = [(g.param((o, i), BF16, F32), g.param((o,), BF16, F32)) for i, o in zip(sizes[:-1], sizes[1:])]
    for i, (w, b) in enumerate(layers):
        if hooks:
            w.set_hook("w%d" % i, hooks)
            b.set_hook("b%d" % i)
        if rs:
            w.set_rs("w%d" % i, 2, rs - 1)
    kept = []
    for step in range(steps):
        g.note("step %d" % step)
        h = x
        for i, (w, b) in enumerate(layers):
            h = h.mm_t(w) + b
            if keep_pre:
                kept.append(h)
            if i < len(layers) - 1:
                h = h.relu()
        loss = h.mse_loss(target)
        loss.forward()
        loss.backward(1.0)
        for w, b in layers:
            if steps > 1:
                w.sgd(momentum=0.9, master=True)
            if zero:
                w.zero_grad()
                b.zero_grad()


for _level in range(4):
    SCENARIOS["mlp/level%d" % _level] = lambda g, _l=_level: _mlp(g, _l)
SCENARIOS["mlp/level1_two_multi_sgd_steps"] = lambda g: _mlp(g, 1, steps=2)
SCENARIOS["mlp/level2_pre_activation_held"] = lambda g: _mlp(g, 2, keep_pre=True)
SCENARIOS["mlp/level3_colsum_unsupported"] = lambda g: _mlp(g, 3, fail="nk_gemm_relu_bwd_colsum")
SCENARIOS["mlp/level2_hooks_row_chunks"] = lambda g: _mlp(g, 2, hooks=2)
SCENARIOS["mlp/level2_rs_push"] = lambda g: _mlp(g, 2, rs=1)
SCENARIOS["mlp/level2_rs_accumulating_multi_sgd"] = lambda g: _mlp(g, 2, steps=2, rs=2, zero=False)
SCENARIOS["mlp/level1_rs_and_hooks"] = lambda g: _mlp(g, 1, rs=2, hooks=2)


# ---- Conv2d (+ bias) (+ ReLU)
def _conv(g, level=1, seed_on_conv=False, input_diff=False, repeat=1, input_grad=None):
    g.fusion(level)
    k = g.param((8, 3, 3, 3), BF16, F32)
    b = g.param((8, 1, 1), BF16, F32)
    x = g.param((2, 3, 10, 10), BF16, input_grad) if input_diff else g.leaf((2, 3, 10, 10), BF16)
    y = k.conv(x.pad(1, 1)) + b
    if seed_on_conv:
        out = y
    else:
        out = y.relu().flatten().mse_loss(g.leaf((2, 800), BF16))
    out.forward()
    for r in range(repeat):
        g.note("backward %d" % r)
        out.backward(1.0)
    for v in (k, b, x):
        if g.lib.nkg_is_diff(v.h):
            v.grad_ptr()


SCENARIOS["conv/bias_relu_loss"] = lambda g: _conv(g)
SCENARIOS["conv/bias_relu_loss_level0"] = lambda g: _conv(g, level=0)
SCENARIOS["conv/seed_on_conv"] = lambda g: _conv(g, seed_on_conv=True)
SCENARIOS["conv/seed_on_conv_input_diff"] = lambda g: _conv(g, seed_on_conv=True, input_diff=True)
SCENARIOS["conv/input_diff_loss"] = lambda g: _conv(g, input_diff=True)
SCENARIOS["conv/input_diff_f32_grad"] = lambda g: _conv(g, input_diff=True, input_grad=F32)
SCENARIOS["conv/repeated_backward_level1"] = lambda g: _conv(g, seed_on_conv=True, repeat=3)


@scenario("repeated_backward/level1")
def _repeated_level1(g):
    x = g.leaf((8, 12))
    w, b = g.param((10, 12)), g.param((10,))
    w2 = g.param((4, 10))
    z = (x.mm_t(w) + b).relu().mm_t(w2)
    s = z.sum()
    s.forward()
    for r in range(3):
        g.note("backward %d" % r)
        s.backward(1.0)
        w.grad_ptr()
        b.grad_ptr()
        w2.grad_ptr()


@scenario("repeated_backward/level2_error")
def _repeated_level2(g):
    g.fusion(2)
    x = g.leaf((8, 12), BF16)
    w1, b1 = g.param((16, 12), BF16), g.param((16,), BF16)
    w2, b2 = g.param((4, 16), BF16), g.param((4,), BF16)
    s = ((x.mm_t(w1) + b1).relu().mm_t(w2) + b2).sum()
    s.forward()
    s.backward(1.0)
    g.expect_error(s.backward, 1.0)


@scenario("grad_state/zero_no_with")
def _grad_state(g):
    x = g.leaf((3, 6))
    w = g.param((4, 6))
    y = x.mm_t(w).relu()
    s = y.sum()
    s.forward()
    s.backward(1.0)
    w.grad_ptr()
    y.grad_ptr("intermediate")
    w.zero_grad()
    w.grad_ptr("after zero_grad")
    s.backward(2.0)
    w.zero_grad()
    s.backward(1.0)
    s.no_grad()
    w.grad_ptr("after no_grad")
    g.expect_error(s.backward, 1.0)
    s.with_grad()
    w.grad_ptr("after with_grad")
    s.forward()
    s.backward(1.0)
    w.grad_ptr()
    y.zero_grad()
    g.expect_error(x.zero_grad)
    g.expect_error(x.no_grad)
    g.expect_error(x.with_grad)


@scenario("grad_state/caller_owned_gradient")
def _caller_owned(g):
    gp = C.c_void_p(g.ext(4 * 6 * 4))
    x = g.leaf((3, 6))
    w = g.leaf((4, 6)).requires_grad(None, gp)
    w.describe("w")
    w.grad_ptr()
    s = x.mm_t(w).sum()
    s.forward()
    s.backward(1.0)
    w.zero_grad()
    s.backward(1.0)
    w.no_grad()
    w.grad_ptr("after no_grad")
    w.with_grad()
    w.grad_ptr("after with_grad")
    s.backward(1.0)
    w.forward()
    w.backward(3.0)          # the seed is written straight into caller-visible memory


@scenario("grad_state/leaf_seed_and_clone")
def _leaf_seed(g):
    w = g.param((4, 6))
    w.forward()
    w.backward(2.0)
    w.grad_ptr()
    c = w.clone()
    c.describe("clone")
    c.backward(1.0)
    w.zero_grad()
    w.grad_ptr()
    e = g.external((5, 3))
    e.describe("external")
    e.data_ptr()
    ed = e.requires_grad(F32)
    s = (ed * ed).sum()
    s.forward()
    s.backward(1.0)
    ed.grad_ptr()


@scenario("views/flatten_unsqueeze")
def _views(g):
    x = g.param((2, 3, 4))
    f = x.flatten()
    f.describe("flatten")
    u = x.unsqueeze(0)
    u.describe("unsqueeze")
    s = f.mm_t(g.leaf((5, 12))).sum() + u.sum()
    s.forward()
    s.backward(1.0)
    x.grad_ptr()
    f.grad_ptr("flatten grad")
    u.grad_ptr("unsqueeze grad")
    v = g.leaf((2, 3)).unsqueeze(2)
    v.describe("var view")
    v.data_ptr()


@scenario("cat/mixed_and_repeated")
def _cat_mixed(g):
    x = g.param((2, 3))
    y = g.param((2, 3), F32, BF16)
    v = g.leaf((2, 3))
    empty = g.param((2, 0))
    c = x.cat([v, x, y, empty, x], 1)
    s = x.stack([v, y, x], 1)
    out = c.sum() + s.mean()
    _run(g, out, x, y, empty)
    cv = v.cat([v], 0)
    cv.describe("var cat")
    w = g.param((3, 2))
    a = x.mm(w) + g.param((2,))             # its gradient is aliased by the peephole
    ca = a.cat([a, x.mm(w)], 0).sum()
    _run(g, ca, x, w)
    z = g.param((0, 3)).cat([g.leaf((0, 3))], 0)
    z.describe("empty")
    z.forward()
    z.backward(1.0)


def _rnn(g, lstm, steps=2, hooks=False, state_diff=False, dtype=BF16):
    N, I, H = 4, 8, 16
    G = (4 if lstm else 3) * H
    w_ih, w_hh = g.param((G, I), dtype, F32), g.param((G, H), dtype, F32)
    b_ih, b_hh = g.param((G,), dtype, F32), g.param((G,), dtype, F32)
    if hooks:
        w_ih.set_hook("w_ih")
        b_hh.set_hook("b_hh")
        w_hh.set_rs("w_hh", 2, 0)
    h = g.param((N, H), dtype, F32) if state_diff else g.leaf((N, H), dtype)
    c = g.param((N, H), dtype, F32) if state_diff else g.leaf((N, H), dtype)
    h0, c0 = h, c
    xs = [g.leaf((N, I), dtype) for _ in range(steps)]
    for x in xs:
        if lstm:
            c, h = g.lstm(x, c, h, w_ih, w_hh, b_ih, b_hh)
        else:
            h = g.gru(x, h, w_ih, w_hh, b_ih, b_hh)
    h.describe("h")
    loss = h.mean()
    loss.forward()
    loss.backward(1.0)
    for v in (w_ih, w_hh, b_ih, b_hh):
        v.grad_ptr()
    if state_diff:
        h0.grad_ptr("h0")
        if lstm:
            c0.grad_ptr("c0")


for _cell in ("lstm", "gru"):
    _l = _cell == "lstm"
    SCENARIOS["rnn/%s_hooks" % _cell] = lambda g, _l=_l: _rnn(g, _l, hooks=True)
    SCENARIOS["rnn/%s_state_diff" % _cell] = lambda g, _l=_l: _rnn(g, _l, state_diff=True)


@scenario("rnn/lstm_both_outputs")
def _lstm_both(g):
    N, I, H = 2, 4, 8
    ws = [g.param(s) for s in ((4 * H, I), (4 * H, H), (4 * H,), (4 * H,))]
    c, h = g.lstm(g.leaf((N, I)), g.param((N, H)), g.param((N, H)), *ws)
    c.describe("c")
    loss = c.sum() + h.sum()
    loss.forward()
    loss.backward(1.0)
    c2, h2 = g.lstm(g.leaf((N, I)), g.leaf((N, H)), g.leaf((N, H)), *[g.leaf(s) for s in ((4 * H, I), (4 * H, H),
                                                                                             (4 * H,), (4 * H,))])
    c2.describe("var c")
    h2.forward()


@scenario("errors")
def _errors(g):
    E, L = g.expect_error, g.lib
    a, b = g.param((4, 6)), g.param((6, 5))
    a16 = g.leaf((6, 5), BF16)
    other = g.leaf((6, 5), F32, g.other_ctx)
    out = C.c_void_p()
    ck = g.ck
    E(lambda: g.leaf((1,) * 7))
    E(lambda: g.leaf((2,), 5))
    E(lambda: ck(L.nkg_leaf(None, 1, _i64s((2,)), 0, C.byref(out))))
    E(lambda: ck(L.nkg_leaf_external(g.ctx, 1, _i64s((2,)), 0, None, C.byref(out))))
    E(lambda: ck(L.nkg_requires_grad(None, -1, None, C.byref(out))))
    E(lambda: ck(L.nkg_clone(None, C.byref(out))))
    E(lambda: ck(L.nkg_forward(None)))
    E(lambda: ck(L.nkg_backward(None, 1.0)))
    for name in ("nkg_mm", "nkg_mm_t", "nkg_add", "nkg_sub", "nkg_mul", "nkg_div", "nkg_mv", "nkg_vm", "nkg_vv"):
        E(lambda: ck(getattr(L, name)(a.h, None, C.byref(out))))
    for name in ("nkg_relu", "nkg_sum", "nkg_mean", "nkg_flatten", "nkg_transpose", "nkg_neg", "nkg_exp"):
        E(lambda: ck(getattr(L, name)(None, C.byref(out))))
    E(lambda: ck(L.nkg_softmax(None, 0, C.byref(out))))
    E(lambda: ck(L.nkg_unsqueeze(None, 0, C.byref(out))))
    E(lambda: ck(L.nkg_mse_loss(a.h, None, 0, C.byref(out))))
    E(lambda: ck(L.nkg_pad(None, 1, 1, 0.0, C.byref(out))))
    E(lambda: ck(L.nkg_pad_mode(a.h, 1, None, 0, 0.0, C.byref(out))))
    E(lambda: ck(L.nkg_convolution(None, a.h, 1, 1, 1, 1, 1, C.byref(out))))
    E(lambda: ck(L.nkg_convolution_nd(a.h, a.h, 1, None, _i64s((1,)), 1, C.byref(out))))
    E(lambda: ck(L.nkg_chunks(None, 1, _i64s((1,)), 0, None, C.byref(C.c_int()))))
    E(lambda: ck(L.nkg_unary(a.h, 9, 0, C.byref(out))))
    # operand checks shared by several recorders (the other validation messages are unchanged source lines)
    E(lambda: a.mm(a16))
    E(lambda: a.mm(other))
    E(lambda: a.mm_t(a16))
    E(lambda: a + a16)
    E(lambda: a - other)
    x4, x3 = g.leaf((2, 4, 8, 8)), g.leaf((2, 4, 8))
    E(lambda: g.leaf((4, 1, 3, 3)).conv(x4, (1, 1), (1, 1), 3))
    E(lambda: g.leaf((3, 2, 3, 3)).conv(x4, (1, 1), (1, 1), 2))
    E(lambda: g.leaf((4, 3, 3, 3)).conv(x4))
    E(lambda: g.leaf((4, 1, 3)).conv_nd(x3, (1,), (1,), 3))
    E(lambda: g.leaf((3, 2, 3)).conv_nd(x3, (1,), (1,), 2))
    E(lambda: g.leaf((4, 3, 3)).conv_nd(x3, (1,), (1,)))
    # concatenation
    E(lambda: ck(L.nkg_cat(None, 1, 0, C.byref(out))))
    E(lambda: ck(L.nkg_stack((C.c_void_p * 2)(a.h.value, None), 2, 0, C.byref(out))))
    # recurrent cells
    N, I, H = 2, 3, 4
    x, h, c = g.leaf((N, I)), g.leaf((N, H)), g.leaf((N, H))
    ws = [g.leaf(s) for s in ((4 * H, I), (4 * H, H), (4 * H,), (4 * H,))]
    E(lambda: g.lstm(x, c, h, None, *ws[1:]))
    E(lambda: g.lstm(x, None, h, *ws))
    E(lambda: ck(L.nkg_lstm_cell(x.h, c.h, h.h, *[w.h for w in ws], None, C.byref(out))))
    E(lambda: ck(L.nkg_gru_cell(x.h, h.h, *[w.h for w in ws], None)))
    # execution and state on the wrong kind of variable
    E(lambda: g.leaf((2,)).backward(1.0))
    y = a.mm(b)
    E(lambda: y.backward(1.0))
    E(lambda: g.leaf((2,)).set_hook("v"))
    E(lambda: g.leaf((2,)).set_rs("v", 2, 0))
    E(lambda: ck(L.nkg_set_grad_rs(a.h, 9, 0, None, None, None)))
    E(lambda: ck(L.nkg_set_grad_rs(a.h, 2, 2, (C.c_void_p * 2)(1, 2), None, None)))
    E(lambda: ck(L.nkg_set_grad_rs(a.h, 2, 0, None, None, None)))
    ck(L.nkg_set_grad_rs(a.h, 1, 0, None, None, None))
    g.note("introspection of NULL: %d %d %d %d %d %d" % (
        L.nkg_is_diff(None), L.nkg_ndim(None), L.nkg_dtype(None), L.nkg_grad_dtype(None), L.nkg_history_len(None),
        L.nkg_backward_history_len(None)))
    g.note("shape(NULL) = %d" % L.nkg_shape(None, None))
    g.note("data_ptr(NULL) = %s, grad_ptr(Var) = %s" % (L.nkg_data_ptr(None), L.nkg_grad_ptr(g.leaf((2,)).h)))
