"""Static ABI check: every ctypes declaration (tf_yarn_b200.ops.native + the op modules' native.declare calls) against
the C signature of the function it binds, parsed from ops/csrc.  The kernels are reached through plain C entry points;
a wrong argument count or an int where a pointer is expected would only show up on a GPU -- as memory corruption."""
import ctypes
import glob
import os
import re


from tf_yarn_b200.ops import native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf_yarn_b200", "ops", "csrc")

_C_FN = re.compile(r"^(?:extern \"C\" )?(int|void|long|void\*|uint64_t|size_t|const char\*)\s+(tfy_\w+)\s*\(([^)]*)\)\s*\{",
                   re.M)


def _c_kind(param: str) -> str:
    p = param.strip()
    if "*" in p or "cudaStream_t" in p or "&" in p:
        return "ptr"
    t = re.sub(r"\b(const|unsigned)\b", lambda m: m.group(0), p)
    t = " ".join(t.split()[:-1]) if len(t.split()) > 1 else t          # drop the parameter name
    t = t.replace("const ", "").strip()
    return {"int": "i32", "int32_t": "i32", "float": "f32", "double": "f64", "size_t": "w64", "uint64_t": "w64",
            "uint32_t": "u32", "long long": "w64", "long": "w64", "int64_t": "w64", "bool": "i32"}.get(t, f"struct:{t}")


def _c_signatures():
    sigs = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp"))):
        src = open(path).read()
        src = re.sub(r"//[^\n]*", "", src)
        for m in _C_FN.finditer(src):
            ret, name, params = m.group(1), m.group(2), m.group(3)
            params = [p for p in (q.strip() for q in params.replace("\n", " ").split(",")) if p and p != "void"]
            sigs[name] = (ret, [_c_kind(p) for p in params], os.path.basename(path))
    return sigs


def _py_kind(t) -> str:
    if t in (ctypes.c_void_p, ctypes.c_char_p) or (isinstance(t, type) and issubclass(t, ctypes._Pointer)):
        return "ptr"
    if isinstance(t, type) and issubclass(t, (ctypes.Structure, ctypes.Array)):
        return "ptr" if issubclass(t, ctypes.Array) else f"struct:{t.__name__}"
    return {ctypes.c_int: "i32", ctypes.c_int32: "i32", ctypes.c_float: "f32", ctypes.c_double: "f64",
            ctypes.c_size_t: "w64", ctypes.c_uint64: "w64", ctypes.c_uint32: "u32", ctypes.c_longlong: "w64",
            ctypes.c_long: "w64", ctypes.c_int64: "w64"}[t]


def _py_declarations():
    # importing the op modules runs their native.declare(...) calls
    import tf_yarn_b200.estimator.ps_hbm  # noqa: F401
    import tf_yarn_b200.keras.fastpath  # noqa: F401
    import tf_yarn_b200.ops.gemm  # noqa: F401
    import tf_yarn_b200.parallel.comm  # noqa: F401
    import tf_yarn_b200.parallel.ddp  # noqa: F401
    try:
        import tf_yarn_b200.ops.nn  # noqa: F401
    except ImportError:
        pass

    class Fn:
        argtypes = None
        restype = ctypes.c_int

    class Lib:
        def __init__(self):
            self.fns = {}

        def __getattr__(self, name):
            if name.startswith("tfy_"):
                return self.__dict__["fns"].setdefault(name, Fn())
            raise AttributeError(name)
    lib = Lib()
    native._declare(lib)
    decls = {name: (fn.argtypes, fn.restype) for name, fn in lib.fns.items() if fn.argtypes is not None}
    decls.update({name: (args, restype) for name, (args, restype) in native._EXTRA_DECLS.items()})
    return decls


def test_every_ctypes_declaration_matches_its_c_signature():
    c = _c_signatures()
    py = _py_declarations()
    assert len(py) >= 40 and len(c) >= len(py)
    problems = []
    for name, (argtypes, restype) in sorted(py.items()):
        if name not in c:
            problems.append(f"{name}: declared in Python, not defined in ops/csrc")
            continue
        ret, c_kinds, where = c[name]
        py_kinds = [_py_kind(t) for t in argtypes]
        if py_kinds != c_kinds:
            problems.append(f"{name} ({where}): python {py_kinds} != C {c_kinds}")
        want_ret = {"int": ctypes.c_int, "void": None, "long": ctypes.c_long, "void*": ctypes.c_void_p,
                    "uint64_t": ctypes.c_uint64, "size_t": ctypes.c_size_t, "const char*": ctypes.c_char_p}[ret]
        if restype is not want_ret and not (want_ret in (ctypes.c_uint64, ctypes.c_size_t)
                                            and restype in (ctypes.c_uint64, ctypes.c_size_t)):
            problems.append(f"{name} ({where}): python restype {restype} != C {ret}")
    assert not problems, "\n".join(problems)


def test_the_parser_sees_the_functions_it_should():
    c = _c_signatures()
    for must in ("tfy_allreduce", "tfy_fused_step", "tfy_gemm_bf16", "tfy_gemm2_bf16", "tfy_dense_bwd", "tfy_ps_push",
                 "tfy_ps_gather_gemm", "tfy_reducer_create", "tfy_symm_open"):
        assert must in c, must
    assert c["tfy_allreduce"][1] == ["ptr", "i32", "i32", "w64", "w64", "f32", "ptr", "i32", "i32", "ptr"]


def test_every_native_call_in_the_package_is_declared():
    """A function called through ctypes WITHOUT argtypes gets Python ints converted to C int: a device pointer would be
    truncated to 32 bits.  Every `.tfy_*(` call site of the package must therefore be a declared function (or one of
    the few argument-less / lazily declared ones)."""
    declared = set(_py_declarations())
    lazily = {"tfy_memcpy_async": [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]}   # engine._capture
    no_args = {"tfy_symm_last_error"}
    kv_lib = {"tfy_kv_start", "tfy_kv_stop", "tfy_kv_port"}                 # libtfy_kv.so, declared in kv/__init__.py
    called = set()
    for path in glob.glob(os.path.join(ROOT, "tf_yarn_b200", "**", "*.py"), recursive=True):
        called |= set(re.findall(r"\.(tfy_\w+)\(", open(path).read()))
    unknown = sorted(called - declared - set(lazily) - no_args - kv_lib)
    assert not unknown, unknown
    c = _c_signatures()
    for name, argtypes in lazily.items():
        assert [_py_kind(t) for t in argtypes] == c[name][1], name
    src = open(os.path.join(ROOT, "tf_yarn_b200", "keras", "engine.py")).read()
    assert 'native.declare("tfy_memcpy_async", [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p])' in src


def test_every_kernel_launched_with_programmatic_dependent_launch_waits_for_its_dependency():
    """A kernel launched with the programmatic-stream-serialisation attribute may start before its predecessor has
    finished; it is only correct if it executes griddepcontrol.wait (tfy_pdl_sync / tfy_pdl_wait) before touching
    global memory.  Every kernel passed to tfy_launch_pdl / tfy_launch_pdl_if must contain that wait, preceded only by
    a prologue that does not dereference its global-memory arguments."""
    launched = {}
    sources = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        src = open(path).read()
        sources[path] = src
        for m in re.finditer(r"tfy_launch_pdl(?:_if)?\((?:[^()]*\(\)[^(]*?)*?\(\s*(tfy_\w+)", src):
            launched.setdefault(m.group(1), path)
    assert len(launched) >= 14, sorted(launched)
    for kernel, path in sorted(launched.items()):
        src = sources[path]
        m = re.search(r"__global__[^;{]*?\b" + re.escape(kernel) + r"\s*\(", src)
        assert m, (kernel, path)
        body_start = src.index("{", m.end())
        depth, i = 0, body_start
        while True:                                             # matching brace of the kernel body
            ch = src[i]
            depth += ch == "{"
            depth -= ch == "}"
            if depth == 0:
                break
            i += 1
        body = re.sub(r"//[^\n]*", "", src[body_start:i])
        waits = [body.find(w) for w in ("tfy_pdl_sync()", "tfy_pdl_wait()") if w in body]
        assert waits, f"{kernel} ({os.path.basename(path)}) is launched with PDL but never waits for its dependency"
        prologue = body[:min(waits)]
        # the prologue may set up shared memory, barriers and prefetch tensor maps / this kernel's own state
        # (tfy_tma_*: the TMA load / store helpers of tfy_tma.cuh)
        for forbidden in ("tfy_ld16(", "__ldg(", "__ldcg(", "atomicAdd(", "tfy_st16(", "red_add", "cp.async.bulk.tensor",
                          "tfy_tma_"):
            assert forbidden not in prologue, (kernel, forbidden)
