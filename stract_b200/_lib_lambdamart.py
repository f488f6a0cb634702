"""ctypes prototypes of the LambdaMART entry points (include/stract_b200_lambdamart.h)."""
import ctypes as C

SIGNAL_ENUM_COUNT = 46   # SB200_SIGNAL_ENUM_COUNT


class LambdaMARTInfo(C.Structure):
    _fields_ = [("n_trees", C.c_uint32), ("n_features", C.c_uint32), ("n_internal", C.c_uint64), ("n_leaves", C.c_uint64),
                ("max_depth", C.c_uint32), ("_pad", C.c_uint32), ("device_bytes", C.c_uint64)]


class LambdaMARTStats(C.Structure):
    _fields_ = [("docs", C.c_uint64), ("ms", C.c_float), ("kernel_ms", C.c_float)]


def proto(L, f):
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    f("sb200_lambdamart_load", i32, C.c_char_p, u64, C.POINTER(vp))
    f("sb200_lambdamart_destroy", None, vp)
    f("sb200_lambdamart_get_info", i32, vp, C.POINTER(LambdaMARTInfo))
    f("sb200_lambdamart_features", i32, vp, vp, u32)
    f("sb200_lambdamart_predict", i32, vp, vp, u64, vp, C.POINTER(LambdaMARTStats))
