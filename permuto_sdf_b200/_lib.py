"""ctypes binding of libpsdf_b200.so, generated from include/psdf_b200.h.

The prototypes are parsed from the header so the Python side can never drift from the C ABI; the CPU test
suite uses `declared_symbols()` to check that the built library exports every declared entry point.
There is no fallback: if the library is missing, or a call is made without a CUDA device, this raises.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "psdf_b200.h")
LIB_PATH = os.path.join(_HERE, "libpsdf_b200.so")

_CTYPES = {
    "int": ctypes.c_int,
    "float": ctypes.c_float,
    "long long": ctypes.c_longlong,
    "uint64_t": ctypes.c_uint64,
    "void*": ctypes.c_void_p,
}


def _parse_header(path=HEADER):
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"//[^\n]*", " ", src)
    macros = dict(re.findall(r"#define\s+(PSDF_RSP)\s+([^\n]+)", src))
    src = re.sub(r"#[^\n]*", " ", src)
    for k, v in macros.items():
        src = src.replace(k, v)
    protos = {}
    for ret, name, args in re.findall(r"\b(int|long long)\s+(psdf_\w+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        arglist = []
        args = " ".join(args.split())
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                m = re.match(r"(const\s+)?([\w ]+?)\s*(\*?)\s*(\w+)(\[\d+\])?$", a)
                if not m:
                    raise RuntimeError("cannot parse argument %r of %s" % (a, name))
                const, base, ptr, aname, arr = m.groups()
                base = base.strip()
                if arr:
                    kind = "float" + arr           # small host array, e.g. float[3]
                elif ptr:
                    kind = "void*" if base == "void" else "ptr:" + base
                else:
                    kind = base
                arglist.append((aname, kind))
        protos[name] = (ret, arglist)
    return protos


PROTOS = _parse_header()


def declared_symbols():
    return sorted(PROTOS)


_lib = None
_NON_STATUS = ("psdf_abi_version", "psdf_device_ok")


def load_library(path=LIB_PATH):
    """dlopen the in-tree CUDA library and attach argtypes. Fails loudly when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise RuntimeError(
            "permuto_sdf_b200: %s not found. Build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "There is no CPU or PyTorch fallback for this path." % path)
    lib = ctypes.CDLL(path)
    for name, (ret, args) in PROTOS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = _CTYPES[ret]
        at = []
        for _, kind in args:
            if kind.startswith("float["):
                at.append(ctypes.c_float * int(kind[6:-1]))
            elif kind.startswith("ptr:") or kind == "void*":
                at.append(ctypes.c_void_p)
            else:
                at.append(_CTYPES[kind])
        fn.argtypes = at
    _lib = lib
    return lib


_DT = None


def _dtypes():
    global _DT
    if _DT is None:
        import torch
        _DT = {"float": (torch.float32,), "int": (torch.int32,), "uint8_t": (torch.uint8, torch.bool), "uint64_t": (torch.int64, torch.uint64),
               "long long": (torch.int64,), "double": (torch.float64,)}
    return _DT


def call(name, *args):
    """Invoke a C-ABI entry point. torch tensors are passed as device pointers (checked: CUDA, contiguous,
    dtype); None -> NULL; n-sequences -> float[n]; the trailing `stream` argument is filled in automatically
    with torch's current stream when omitted."""
    import torch
    lib = load_library()
    ret, protos = PROTOS[name]
    # launch on the device that holds the tensors (and on ITS current stream), not on whatever device happens to be current
    for a in args:
        if isinstance(a, torch.Tensor) and a.is_cuda:
            if a.device.index != torch.cuda.current_device():
                with torch.cuda.device(a.device):
                    return call(name, *args)
            break
    if len(args) == len(protos) - 1 and protos and protos[-1][0] == "stream":
        args = args + (torch.cuda.current_stream().cuda_stream,)
    if len(args) != len(protos):
        raise TypeError("%s expects %d arguments, got %d" % (name, len(protos), len(args)))
    conv = []
    for (aname, kind), a in zip(protos, args):
        if kind.startswith("ptr:"):
            if a is None:
                conv.append(None)
            elif isinstance(a, torch.Tensor):
                if not a.is_cuda:
                    raise RuntimeError("%s(%s): tensor must live on a CUDA device (no CPU path exists)" % (name, aname))
                if not a.is_contiguous():
                    raise RuntimeError("%s(%s): tensor must be contiguous" % (name, aname))
                if a.dtype not in _dtypes()[kind[4:]]:
                    raise RuntimeError("%s(%s): expected %s tensor, got %s" % (name, aname, kind[4:], a.dtype))
                conv.append(a.data_ptr())
            else:
                conv.append(int(a))
        elif kind.startswith("float["):
            n = int(kind[6:-1])
            conv.append((ctypes.c_float * n)(*[float(a[i]) for i in range(n)]))
        elif kind == "void*":
            conv.append(a)
        elif kind == "float":
            conv.append(float(a))
        else:
            conv.append(int(a))
    if _STATS is not None:
        _STATS["calls"][name] = _STATS["calls"].get(name, 0) + 1
        if name in _UNITS_FN:                            # samples processed by a multi-set launch
            u = _STATS.setdefault("units", {})
            u[name] = u.get(name, 0) + _UNITS_FN[name](args)
        elif args and isinstance(args[0], int):          # leading count argument (samples / rays) of the entry point
            u = _STATS.setdefault("units", {})
            u[name] = u.get(name, 0) + int(args[0])
        if name in _KERNELS_FN:
            _STATS["extra"] = _STATS.get("extra", 0) + _KERNELS_FN[name](args) - 1
        if _STATS["events"] is not None:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            rc = getattr(lib, name)(*conv)
            e.record()
            _STATS["events"].setdefault(name, []).append((s, e))
        else:
            rc = getattr(lib, name)(*conv)
    else:
        rc = getattr(lib, name)(*conv)
    if ret == "int" and rc != 0 and name not in _NON_STATUS:
        raise RuntimeError("%s failed with code %d" % (name, rc))
    return rc


# ---- instrumentation used by bench.py: count C-ABI calls / kernel launches and time them with CUDA events on the
# launching stream. Kernel launches per entry point (the rest launch exactly one kernel):
_KERNELS_PER_CALL = {"psdf_packed_compact_scan": 2, "psdf_vr_combine_uniform_samples_with_imp": 3,
                     "psdf_sdf_fused_backward": 2, "psdf_sdf_fused_backward_multi": 2,      # tensor-core kernel + lattice scatter
                     "psdf_sdf_fused_backward_multi_dim": 2,
                     "psdf_bg_fused_backward": 2, "psdf_nerf_fused_backward": 2}


# entry point -> launches as a function of its arguments: the deterministic encoding backward adds the fixed-point flush when it has a
# lattice output
_KERNELS_FN = {"psdf_enc_backward_fx": lambda a: 2 if a[13] is not None else 1,
               "psdf_enc_double_backward_fx": lambda a: 2 if a[14] is not None else 1}
_UNITS_FN = {"psdf_sdf_fused_forward_multi": lambda a: int(a[10]) + int(a[15]),
             "psdf_sdf_fused_forward_dim": lambda a: int(a[1]),
             "psdf_sdf_sphere_trace_dim": lambda a: int(a[4]),
             "psdf_sdf_fused_backward_multi": lambda a: int(a[10]) + int(a[15]) + int(a[20]),
             "psdf_sdf_fused_backward_multi_dim": lambda a: int(a[11]) + int(a[16]) + int(a[21])}
_STATS = None
LAST_UNITS = {}        # {entry point: sum of its leading count argument} of the last stats window


def stats_begin(with_events=False):
    global _STATS
    _STATS = {"calls": {}, "events": {} if with_events else None}


def stats_pause():
    """suspend the current statistics window (a nested window may run in between); -> token for stats_resume"""
    global _STATS
    st, _STATS = _STATS, None
    return st


def stats_resume(token):
    global _STATS
    _STATS = token


def stats_add_launches(n):
    """kernels of this library launched outside `call` (a replayed graph) inside the current window"""
    if _STATS is not None:
        _STATS["extra"] = _STATS.get("extra", 0) + int(n)


def stats_end():
    """-> (calls per entry point, kernel launches, {name: (n, total_ms)} if events were recorded)"""
    global _STATS
    global LAST_UNITS
    st, _STATS = _STATS, None
    LAST_UNITS = st.get("units", {})
    launches = sum(n * _KERNELS_PER_CALL.get(k, 1) for k, n in st["calls"].items()) + st.get("extra", 0)
    times = {}
    if st["events"] is not None:
        import torch
        torch.cuda.synchronize()
        for k, evs in st["events"].items():
            times[k] = (len(evs), sum(s.elapsed_time(e) for s, e in evs))
    return st["calls"], launches, times
