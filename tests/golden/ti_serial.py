"""A serial stand-in for the sliver of Taichi that the reference's gsconverter/processing/gpu_ops.py uses, so
that the REFERENCE'S OWN KERNEL SOURCE (k_means_assign, k_means_update, sor_compute_mean_dists and the host
drivers _kmeans_taichi / filter_sor_gpu around them) can be executed in this container, where the real taichi
wheel cannot be installed.  TEST INFRASTRUCTURE ONLY -- used by make_taichi_goldens.py (which writes
tests/golden/g4_reference_kernels.npz) and by make_taichi_golden_g9.py (tests/golden/g9_reference_stand_in_small.npz).

`install()` puts a module named `taichi` into sys.modules.  Its `@ti.kernel` takes the decorated function's
source text (inspect.getsource), rewrites the AST so that Python's untyped scalars behave like Taichi's
statically typed ones, and runs the body as ordinary Python, one loop iteration after the other.  Nothing of the
kernel is restated here: control flow, operation order, constants, the insertion sort, the hash expression are
whatever the reference file says.  What the shim DOES assert about Taichi (each also stated in SURVEY.md
Appendix A, and each the thing the C oracle assumes as well):

  T1  default_ip = i32, default_fp = f32 (ti.init is called without overrides, gpu_ops.py:14): an integer
      literal, `int(x)` and an `int`-annotated kernel argument are i32; a float literal, `float(x)` and a
      `float`-annotated argument are f32.  Implemented with NumPy scalars: np.int32 / np.float32 arithmetic
      stays in its type (NEP 50), i32 products wrap (two's complement) as they do in Taichi's LLVM/CUDA code.
  T2  `%` on integers is Python's floor-mod (Taichi >= 0.8); with C-style remainder the reference's following
      `if h < 0: h += hash_size` would give the same value, so the result does not depend on this.
  T3  float arithmetic is IEEE round-to-nearest per operation, in source order, no contraction
      (the "strict" reading, SURVEY Appendix A; Taichi's fast_math may contract on a real GPU).
  T4  the outermost `for i in range(N)` of a kernel is a parallel loop whose iterations are independent for
      k_means_assign / sor_compute_mean_dists; for k_means_update's `ti.atomic_add` accumulation the serial
      index order is taken (on a GPU the float atomics land in an unspecified order: the reference's own
      centroids are only reproducible up to that order, north_star tolerance 1e-5 relative).
  T5  ndarray arguments are the caller's NumPy arrays, accessed in place (`a[i, j]`).

Selecting the i64 reading of the probe hash (oracle hash_mode "i64") is NOT offered: under T1 the reference's
expression `(nx * p1) ^ ...` is i32.
"""
from __future__ import annotations

import ast
import inspect
import sys
import textwrap
import types

import numpy as np

_I32 = np.int32
_F32 = np.float32


def _range(*args):
    a = [int(x) for x in args]
    for j in range(*a):
        yield _I32(j)


def _i32cast(x):
    # int(float) truncates toward zero in Taichi as in C; the reference only casts floor() results
    return _I32(int(x))


def _f32cast(x):
    return _F32(x)


def _vector(elems):
    return np.array([_F32(e) for e in elems], dtype=np.float32)


def _floor(x):
    return np.floor(x)        # float32 in, float32 out


def _sqrt(x):
    return np.sqrt(x)         # float32 in, float32 out, correctly rounded


class _Typed(ast.NodeTransformer):
    """Literals -> typed constants (hoisted into the namespace), int()/float()/range() -> typed versions,
    `ti.atomic_add(a[idx], v)` statement -> `a[idx] += v`."""

    def __init__(self):
        self.consts = {}

    def _const(self, value):
        name = f"_k{len(self.consts)}"
        self.consts[name] = value
        return ast.Name(id=name, ctx=ast.Load())

    def visit_Constant(self, node):
        v = node.value
        if isinstance(v, bool) or v is None or isinstance(v, str):
            return node
        if isinstance(v, int):
            return ast.copy_location(self._const(_I32(v)), node)
        if isinstance(v, float):
            return ast.copy_location(self._const(_F32(v)), node)
        return node

    def visit_BinOp(self, node):
        # `[1.0e10] * 50`: a Python-scope list repeat (the argument of ti.Vector), the count stays a Python int
        if isinstance(node.left, ast.List) and isinstance(node.op, ast.Mult) and isinstance(node.right, ast.Constant):
            node.left = self.visit(node.left)
            return node
        return self.generic_visit(node)

    def visit_Call(self, node):
        node = self.generic_visit(node)
        if isinstance(node.func, ast.Name):
            repl = {"int": "_ti_i32cast", "float": "_ti_f32cast", "range": "_ti_range"}.get(node.func.id)
            if repl:
                node.func = ast.Name(id=repl, ctx=ast.Load())
        return node

    def visit_Expr(self, node):
        c = node.value
        if (isinstance(c, ast.Call) and isinstance(c.func, ast.Attribute) and c.func.attr == "atomic_add"
                and isinstance(c.args[0], ast.Subscript)):
            target = self.generic_visit(c.args[0])
            target.ctx = ast.Store()
            aug = ast.AugAssign(target=target, op=ast.Add(), value=self.visit(c.args[1]))
            return ast.copy_location(aug, node)
        return self.generic_visit(node)


def _kernel(fn):
    src = textwrap.dedent(inspect.getsource(fn))
    tree = ast.parse(src)
    fdef = tree.body[0]
    assert isinstance(fdef, ast.FunctionDef)
    kinds = []
    for a in fdef.args.args:
        ann = a.annotation
        kinds.append(ann.id if isinstance(ann, ast.Name) else "ndarray")   # `int`, `float`, else ti.types.ndarray()
        a.annotation = None
    fdef.decorator_list = []
    tr = _Typed()
    fdef.body = [tr.visit(s) for s in fdef.body]
    ast.fix_missing_locations(tree)
    ns = dict(fn.__globals__)
    ns.update(tr.consts)
    ns.update(_ti_i32cast=_i32cast, _ti_f32cast=_f32cast, _ti_range=_range)
    exec(compile(tree, f"<ti_serial:{fn.__name__}>", "exec"), ns)
    body = ns[fdef.name]

    def launch(*args):
        assert len(args) == len(kinds)
        conv = []
        for a, kind in zip(args, kinds):
            if kind == "int":
                assert -2**31 <= int(a) < 2**31
                conv.append(_I32(a))
            elif kind == "float":
                conv.append(_F32(a))
            else:
                assert isinstance(a, np.ndarray)
                conv.append(a)
        with np.errstate(over="ignore"):   # i32 products wrap (T1)
            body(*conv)

    launch.__name__ = fn.__name__
    launch.__ti_serial_source__ = ast.unparse(tree)
    return launch


def install():
    """Insert the stand-in as `taichi` (idempotent); returns the module."""
    m = sys.modules.get("taichi")
    if m is not None and getattr(m, "__ti_serial__", False):
        return m
    m = types.ModuleType("taichi")
    m.__ti_serial__ = True
    m.kernel = _kernel
    m.gpu = "gpu"
    m.cpu = "cpu"
    m.init = lambda *a, **k: None
    m.sync = lambda: None
    m.floor = _floor
    m.sqrt = _sqrt
    m.Vector = _vector
    m.types = types.SimpleNamespace(ndarray=lambda *a, **k: "ndarray")
    m.i32, m.f32 = _I32, _F32
    sys.modules["taichi"] = m
    return m


def import_reference_gpu_ops(ref_root="/root/reference"):
    """Load the reference's gpu_ops.py, unmodified, as a stand-alone module with the stand-in as `taichi`.
    (Loaded by file path so that the package's other imports -- plyfile etc. -- are not needed.)"""
    import importlib.util
    install()
    path = f"{ref_root}/gsconverter/processing/gpu_ops.py"
    spec = importlib.util.spec_from_file_location("_ref_gpu_ops_ti_serial", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.HAS_TAICHI is True
    return mod
