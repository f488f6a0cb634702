"""ctypes loader of libstract_b200.so.  Fails loudly when the CUDA library is missing: the product
path has no CPU fallback."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libstract_b200.so")
_LIB = None


class Sb200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"sb200 error {code}: {msg}")
        self.code = code


class GraphInfo(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("n_edges_input", C.c_uint64), ("n_edges_kept", C.c_uint64),
                ("n_edges_local", C.c_uint64), ("row_begin", C.c_uint64), ("row_end", C.c_uint64),
                ("hbm_bytes", C.c_uint64), ("stage_ms", C.c_double)]


class KernelProf(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("launches", C.c_uint64), ("ms", C.c_double), ("alg_bytes", C.c_double)]


IPC_BLOB_BYTES = 384  # SB200_IPC_BLOB_BYTES


class IterStats(C.Structure):
    _fields_ = [("t", C.c_uint32), ("mode", C.c_uint32), ("n_changed", C.c_uint64),
                ("edges_active", C.c_uint64), ("ms", C.c_float)]


def lib():
    """The loaded C-ABI library (raises if it has not been built: run __graft_entry__.build())."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(_SO):
        raise ImportError(f"{_SO} is missing -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(stract_b200 has no CPU fallback)")
    _LIB = declare(C.CDLL(_SO))
    return _LIB


def declare(L):
    """Attach the C-ABI prototypes to a loaded library handle (lib() does this for libstract_b200.so; the CPU
    emulation tests do it for their own build of the same sources)."""
    vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int

    def f(name, res, *args):
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = list(args)

    f("sb200_last_error", C.c_char_p)
    f("sb200_version", C.c_char_p)
    f("sb200_kernel_launch_count", u64)
    f("sb200_release_cached_memory", i32, i32)
    f("sb200_graph_create", i32, vp, vp, vp, vp, vp, u64, u64, i32, i32, i32, C.POINTER(vp))
    f("sb200_graph_destroy", None, vp)
    f("sb200_graph_get_info", i32, vp, C.POINTER(GraphInfo))
    f("sb200_hyperball_set_policy", i32, vp, C.c_double, C.c_double, i32)
    f("sb200_hyperball_reset", i32, vp)
    f("sb200_hyperball_step", i32, vp, C.POINTER(IterStats))
    f("sb200_hyperball_run", i32, vp, u32, C.POINTER(u32), C.POINTER(IterStats), u32)
    f("sb200_hyperball_last_run_ms", i32, vp, C.POINTER(C.c_float))
    f("sb200_hyperball_set_profiling", i32, vp, i32)
    f("sb200_hyperball_get_profile", i32, vp, C.POINTER(KernelProf), u32, C.POINTER(u32))
    f("sb200_synth_edges", i32, i32, u64, u64, u64, u64, i32, i32, vp, vp, vp, vp, vp)
    f("sb200_hyperball_result", i32, vp, vp, vp, vp, u64, C.POINTER(u64))
    f("sb200_hyperball_ranked", i32, vp, i32, vp, vp, vp, u64, C.POINTER(u64))
    f("sb200_hyperball_registers", i32, vp, u64, u64, vp)
    f("sb200_hyperball_kahan", i32, vp, u64, u64, vp, vp)
    f("sb200_graph_node_ids", i32, vp, u64, u64, vp, vp)
    f("sb200_hyperball_exchange_ptrs", i32, vp, C.POINTER(vp), C.POINTER(u64), C.POINTER(vp), C.POINTER(u64))
    f("sb200_graph_row_ranges", i32, vp, C.POINTER(u64))
    f("sb200_hyperball_exchange_done", i32, vp, u64)
    f("sb200_hyperball_ipc_export", i32, vp, vp)
    f("sb200_hyperball_ipc_import", i32, vp, vp)
    f("sb200_hyperball_p2p_enable", i32, vp, i32)
    f("sb200_hyperball_run_sharded", i32, vp, u32, C.POINTER(u32), C.POINTER(IterStats), u32)
    f("sb200_hyperball_group_link", i32, C.POINTER(vp), i32)
    f("sb200_hyperball_group_run", i32, C.POINTER(vp), i32, u32, C.POINTER(u32), C.POINTER(IterStats), u32)
    f("sb200_graph_ownership", i32, vp, vp, vp)
    f("sb200_graph_distances", i32, vp, vp, vp, vp, u32, u32, u32, i32, vp)
    f("sb200_hyperball_set_option", i32, vp, C.c_char_p, C.c_double)
    f("sb200_inbound_similarity", i32, vp, vp, vp, u32, vp, vp, u32, vp, vp, u32, i32, C.c_double, vp)
    f("sb200_approx_harmonic", i32, vp, vp, vp, u32, u32, u64, vp, vp, vp, u64, C.POINTER(u64))
    f("sb200_hyperball_state_bytes", i32, vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64))
    f("sb200_hyperball_bind_state", i32, vp, vp, vp, vp, vp)
    f("sb200_hyperball_set_publish_targets", i32, vp, i32, vp, vp, vp, vp)
    if hasattr(L, "sb200_betweenness"):   # absent from the CPU emulator library of the HyperBall / BM25 tests
        f("sb200_betweenness", i32, vp, vp, vp, u32, vp, vp, vp, u64, C.POINTER(u64), C.POINTER(u32))
    try:
        from . import _lib_bm25
        _lib_bm25.proto(L, f)
    except ImportError:
        pass
    from . import _lib_lambdamart
    try:
        _lib_lambdamart.proto(L, f)
    except AttributeError:   # a build of a subset of the sources (the CPU emulator library of the BM25 / HyperBall tests)
        pass
    return L


def check(rc):
    if rc != 0:
        raise Sb200Error(rc, lib().sb200_last_error().decode("utf-8", "replace"))


def kernel_launch_count():
    return int(lib().sb200_kernel_launch_count())


def version():
    return lib().sb200_version().decode()
