"""Stract's LambdaMART model (core/src/ranking/models/lambdamart.rs) on the device: the reference's LightGBM text format, parsed
and validated by the library, and a batched predict over a [n_docs][SignalEnum] feature matrix (include/stract_b200_lambdamart.h).

    model = LambdaMART.open("lambdamart.txt")
    scores = model.predict(model.feature_rows(pages))      # pages: ranking_pipeline.Page

predict() gives, bit for bit, LambdaMART::predict: the f64 sum of the trees' leaves in tree order divided by the number of trees.
A model the reference would panic on (or loop forever on) at predict time is refused at load with Sb200Error (SB200_EFORMAT)."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib_lambdamart import SIGNAL_ENUM_COUNT, LambdaMARTInfo, LambdaMARTStats
from .ranking_pipeline import SIGNAL_ENUM

assert len(SIGNAL_ENUM) == SIGNAL_ENUM_COUNT
_ORDINAL = {name: i for i, name in enumerate(SIGNAL_ENUM)}


class LambdaMART:
    """A loaded model.  `features`: the header's SignalEnum names in header order; `n_trees`; `info`: the library's counts."""

    def __init__(self, handle):
        self._h = handle
        L = _lib.lib()
        info = LambdaMARTInfo()
        _lib.check(L.sb200_lambdamart_get_info(self._h, C.byref(info)))
        self.n_trees = int(info.n_trees)
        ords = np.zeros(info.n_features, np.uint32)
        _lib.check(L.sb200_lambdamart_features(self._h, ords.ctypes.data, ords.size))
        self.features = [SIGNAL_ENUM[int(o)] for o in ords]
        self.info = {"n_trees": int(info.n_trees), "n_features": int(info.n_features), "n_internal": int(info.n_internal),
                     "n_leaves": int(info.n_leaves), "max_depth": int(info.max_depth), "device_bytes": int(info.device_bytes)}
        self.last_stats = None

    @classmethod
    def parse(cls, text):
        """LambdaMART::parse of `text` (str or UTF-8 bytes) onto the current CUDA device"""
        data = text.encode("utf-8") if isinstance(text, str) else bytes(text)
        h = C.c_void_p()
        _lib.check(_lib.lib().sb200_lambdamart_load(data, len(data), C.byref(h)))
        return cls(h)

    @classmethod
    def open(cls, path):
        """LambdaMART::open: the file's bytes (invalid UTF-8 is refused like the reference's read_to_string)"""
        with open(path, "rb") as f:
            return cls.parse(f.read())

    def close(self):
        if self._h:
            _lib.lib().sb200_lambdamart_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def feature_rows(pages):
        """The [len(pages)][SignalEnum] f64 matrix of ranking_pipeline.Page signal scores, 0.0 where a page lacks a signal
        (the reference reads SignalCalculation::score with unwrap_or(0.0))"""
        m = np.zeros((len(pages), SIGNAL_ENUM_COUNT))
        for i, p in enumerate(pages):
            for name, (_value, score) in p.signals.items():
                m[i, _ORDINAL[name]] = score
        return m

    def predict(self, matrix):
        """One prediction per row of `matrix`: a float64 numpy array [n][46], or a CUDA float64 torch tensor of that shape, which
        is read in place (the result is then a CUDA tensor on the same device).  Stats of the call in `last_stats`."""
        L = _lib.lib()
        st = LambdaMARTStats()
        if type(matrix).__module__.startswith("torch"):
            import torch
            if not matrix.is_cuda or matrix.dtype != torch.float64 or matrix.dim() != 2 or matrix.shape[1] != SIGNAL_ENUM_COUNT:
                raise ValueError("a torch feature matrix must be a CUDA float64 tensor of shape [n, 46]")
            x = matrix.contiguous()
            out = torch.empty(x.shape[0], dtype=torch.float64, device=x.device)
            torch.cuda.synchronize(x.device)   # the library's stream does not order itself after torch's
            _lib.check(L.sb200_lambdamart_predict(self._h, C.c_void_p(x.data_ptr()), x.shape[0], C.c_void_p(out.data_ptr()),
                                                  C.byref(st)))
        else:
            x = np.ascontiguousarray(matrix, dtype=np.float64)
            if x.ndim != 2 or x.shape[1] != SIGNAL_ENUM_COUNT:
                raise ValueError(f"feature matrix must have shape [n, {SIGNAL_ENUM_COUNT}], got {x.shape}")
            out = np.empty(x.shape[0])
            _lib.check(L.sb200_lambdamart_predict(self._h, x.ctypes.data, x.shape[0], out.ctypes.data, C.byref(st)))
        self.last_stats = {"docs": int(st.docs), "ms": float(st.ms), "kernel_ms": float(st.kernel_ms)}
        return out
