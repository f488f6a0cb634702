"""ctypes prototypes + helpers for the path-2 (BM25) oracle.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(np.uint32, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(np.uint64, flags="C_CONTIGUOUS")
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")


def proto(L, f):
    vp, u32, u64, i32, f32, f64 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_float, C.c_double
    f("orc_id_to_fieldnorm", u32, C.c_uint8)
    f("orc_fieldnorm_to_id", C.c_uint8, u32)
    f("orc_bp4_roundtrip", u64, _u32p, C.c_uint8, _u8p, _u32p)
    f("orc_vint_sorted_encode", u64, _u32p, u32, u32, _u8p)
    f("orc_encode_bitwidth", C.c_uint8, C.c_uint8, i32)
    f("orc_tv_idf", f32, u64, u64)
    f("orc_tv_bm25_weight", None, f32, f32, C.POINTER(f32), _f32p)
    f("orc_tv_bm25_score", f32, f32, _f32p, C.c_uint8, u32)
    f("orc_stract_bm25_weight", None, f32, f32, f32, f32, C.POINTER(f32), _f32p)
    f("orc_stract_bm25_score", f32, f32, _f32p, f32, C.c_uint8, u32)
    f("orc_seg_new", vp, _u8p, u32)
    f("orc_seg_free", None, vp)
    f("orc_seg_avg_fieldnorm", f32, vp)
    f("orc_seg_set_avg_fieldnorm", None, vp, f32)
    f("orc_seg_set_record", None, vp, i32)
    f("orc_tis_write", u64, _u32p, _u64p, _u64p, _u64p, _u64p, u64, vp)
    f("orc_tis_get", None, _u8p, u64, u64, C.POINTER(u32), C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), C.POINTER(u64))
    f("orc_tis_num_terms", u64, _u8p)
    f("orc_bitpack", u64, _u64p, _u8p, u32, _u8p)
    f("orc_extract_bits", u64, _u8p, u64, u64, C.c_uint8)
    f("orc_seg_add_term", u32, vp, _u32p, _u32p, u32)
    f("orc_seg_postings_len", u64, vp)
    f("orc_seg_postings_copy", None, vp, _u8p)
    f("orc_seg_num_terms", u32, vp)
    f("orc_seg_term_info", None, vp, u32, C.POINTER(u64), C.POINTER(u64), C.POINTER(u32))
    f("orc_seg_set_postings", None, vp, _u8p, u64, _u64p, _u64p, _u32p, u32)
    f("orc_bm25_topk", u32, vp, _u32p, _f32p, _f32p, u32, i32, u32, _u32p, _f32p, C.POINTER(u64))
    f("orc_signal_topk", u32, vp, _u32p, _f32p, _f32p, f32, u32, f64, vp, _f64p, u32, u32, u32, _u32p, _f64p, C.POINTER(u64))
    f("orc_bm25_topk_batch", None, vp, _u32p, _f32p, _f32p, u32, i32, u32, u32, i32, _u32p, _f32p, _u32p, _u64p)
    f("orc_signal_topk_batch", None, vp, _u32p, _f32p, _f32p, f32, u32, f64, vp, _f64p, u32, u32, u32, u32, i32, _u32p,
      _f64p, _u32p, _u64p)
    f("orc_multi_signal_topk", u32, u32, vp, vp, _f32p, _f32p, u32, _u8p, _u32p, _f32p, _f32p, vp, u32, _u32p, _u32p, _u32p, _u32p, _f64p,
      vp, u32, _u32p, _f64p, C.POINTER(u64))
    f("orc_topn_f64", u32, _f64p, _u32p, u32, u32, _u32p, _f64p)
    f("orc_cursor_open", vp, vp, u32, f32, _f32p)
    f("orc_cursor_free", None, vp)
    for name in ("doc", "tf", "advance", "last_doc_in_block"):
        f(f"orc_cursor_{name}", u32, vp)
    f("orc_cursor_seek", u32, vp, u32)
    f("orc_cursor_shallow_seek", None, vp, u32)
    for name in ("score", "max_score", "block_max_score"):
        f(f"orc_cursor_{name}", f32, vp)


def _L():
    from .pyoracle import lib
    return lib()


def fieldnorm_to_id(fn):
    return int(_L().orc_fieldnorm_to_id(int(fn)))


def id_to_fieldnorm(i):
    return int(_L().orc_id_to_fieldnorm(int(i)))


FIELDNORM_TABLE = None


def fieldnorm_table():
    global FIELDNORM_TABLE
    if FIELDNORM_TABLE is None:
        FIELDNORM_TABLE = np.array([id_to_fieldnorm(i) for i in range(256)], np.uint32)
    return FIELDNORM_TABLE


def fieldnorms_to_ids(fieldnorms):
    t = fieldnorm_table()
    return (np.searchsorted(t, np.asarray(fieldnorms, np.uint32), side="right") - 1).astype(np.uint8)


def tv_bm25_weight(doc_freq, num_docs, avg_fieldnorm):
    """tantivy Bm25Weight::for_one_term -> (weight f32, cache[256] f32)."""
    L = _L()
    idf = L.orc_tv_idf(int(doc_freq), int(num_docs))
    w = C.c_float(0)
    cache = np.zeros(256, np.float32)
    L.orc_tv_bm25_weight(idf, float(avg_fieldnorm), C.byref(w), cache)
    return np.float32(w.value), cache


def stract_bm25_weight(doc_freq, num_docs, avg_fieldnorm, k1=1.2, b=0.75):
    L = _L()
    idf = L.orc_tv_idf(int(doc_freq), int(num_docs))  # same idf expression (core/src/ranking/bm25.rs:23-27)
    w = C.c_float(0)
    cache = np.zeros(256, np.float32)
    L.orc_stract_bm25_weight(idf, float(avg_fieldnorm), float(k1), float(b), C.byref(w), cache)
    return np.float32(w.value), cache


class Segment:
    """One field of one segment: postings file in tantivy's byte format + fieldnorm ids."""

    def __init__(self, fieldnorm_ids, avg_fieldnorm=None, record_option=1):
        self.fieldnorm_ids = np.ascontiguousarray(fieldnorm_ids, np.uint8)
        self.max_doc = int(self.fieldnorm_ids.size)
        self.L = _L()
        self.h = self.L.orc_seg_new(self.fieldnorm_ids, self.max_doc)
        if avg_fieldnorm is not None:
            self.L.orc_seg_set_avg_fieldnorm(self.h, float(avg_fieldnorm))
        self.record_option = int(record_option)
        self.L.orc_seg_set_record(self.h, self.record_option)

    @property
    def avg_fieldnorm(self):
        return float(self.L.orc_seg_avg_fieldnorm(self.h))

    def add_term(self, docs, tfs):
        docs = np.ascontiguousarray(docs, np.uint32); tfs = np.ascontiguousarray(tfs, np.uint32)
        assert docs.size == tfs.size
        return int(self.L.orc_seg_add_term(self.h, docs, tfs, docs.size))

    def postings_bytes(self):
        n = int(self.L.orc_seg_postings_len(self.h))
        out = np.zeros(max(n, 1), np.uint8)
        self.L.orc_seg_postings_copy(self.h, out)
        return out[:n]

    def term_infos(self):
        n = int(self.L.orc_seg_num_terms(self.h))
        off = np.zeros(n, np.uint64); ln = np.zeros(n, np.uint64); df = np.zeros(n, np.uint32)
        o, l, d = C.c_uint64(), C.c_uint64(), C.c_uint32()
        for t in range(n):
            self.L.orc_seg_term_info(self.h, t, C.byref(o), C.byref(l), C.byref(d))
            off[t], ln[t], df[t] = o.value, l.value, d.value
        return off, ln, df

    def set_postings(self, data, off, ln, df):
        data = np.ascontiguousarray(data, np.uint8)
        self.L.orc_seg_set_postings(self.h, data, data.size, np.ascontiguousarray(off, np.uint64),
                                    np.ascontiguousarray(ln, np.uint64), np.ascontiguousarray(df, np.uint32), len(df))

    def topk(self, terms, weights, caches, mode, k):
        terms = np.ascontiguousarray(terms, np.uint32); weights = np.ascontiguousarray(weights, np.float32)
        caches = np.ascontiguousarray(caches, np.float32).reshape(-1)
        docs = np.zeros(k, np.uint32); scores = np.zeros(k, np.float32); sc = C.c_uint64(0)
        n = self.L.orc_bm25_topk(self.h, terms, weights, caches, terms.size, mode, k, docs, scores, C.byref(sc))
        return docs[:n], scores[:n], sc.value

    def topk_batch(self, terms, weights, caches, mode, k, threads=1):
        terms = np.ascontiguousarray(terms, np.uint32); nq, nt = terms.shape
        weights = np.ascontiguousarray(weights, np.float32); caches = np.ascontiguousarray(caches, np.float32)
        docs = np.zeros((nq, k), np.uint32); scores = np.zeros((nq, k), np.float32)
        n_out = np.zeros(nq, np.uint32); scored = np.zeros(nq, np.uint64)
        self.L.orc_bm25_topk_batch(self.h, terms.reshape(-1), weights.reshape(-1), caches.reshape(-1), nt, mode, k, nq,
                                   threads, docs.reshape(-1), scores.reshape(-1), n_out, scored)
        return docs, scores, n_out, scored

    def _sig(self, signals):
        sigs = [np.ascontiguousarray(s, np.float64) for s in signals]
        arr = (C.c_void_p * max(len(sigs), 1))(*[s.ctypes.data for s in sigs])
        return sigs, arr

    def signal_topk(self, terms, weights, caches, k1, coeff_text, signals, coeffs, k, max_docs=0):
        terms = np.ascontiguousarray(terms, np.uint32); weights = np.ascontiguousarray(weights, np.float32)
        caches = np.ascontiguousarray(caches, np.float32).reshape(-1)
        sigs, arr = self._sig(signals)
        co = np.ascontiguousarray(coeffs, np.float64) if len(sigs) else np.zeros(1, np.float64)
        docs = np.zeros(k, np.uint32); totals = np.zeros(k, np.float64); sc = C.c_uint64(0)
        n = self.L.orc_signal_topk(self.h, terms, weights, caches, float(k1), terms.size, float(coeff_text),
                                   C.cast(arr, C.c_void_p), co, len(sigs), max_docs, k, docs, totals, C.byref(sc))
        return docs[:n], totals[:n], sc.value

    def signal_topk_batch(self, terms, weights, caches, k1, coeff_text, signals, coeffs, k, max_docs=0, threads=1):
        terms = np.ascontiguousarray(terms, np.uint32); nq, nt = terms.shape
        weights = np.ascontiguousarray(weights, np.float32); caches = np.ascontiguousarray(caches, np.float32)
        sigs, arr = self._sig(signals)
        co = np.ascontiguousarray(coeffs, np.float64) if len(sigs) else np.zeros(1, np.float64)
        docs = np.zeros((nq, k), np.uint32); totals = np.zeros((nq, k), np.float64)
        n_out = np.zeros(nq, np.uint32); scored = np.zeros(nq, np.uint64)
        self.L.orc_signal_topk_batch(self.h, terms.reshape(-1), weights.reshape(-1), caches.reshape(-1), float(k1), nt,
                                     float(coeff_text), C.cast(arr, C.c_void_p), co, len(sigs), max_docs, k, nq, threads,
                                     docs.reshape(-1), totals.reshape(-1), n_out, scored)
        return docs, totals, n_out, scored

    def cursor(self, term, weight, cache):
        return Cursor(self, term, weight, cache)

    def close(self):
        if self.h:
            self.L.orc_seg_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def multi_signal_topk(segments, caches, k1s, coefs, slot_field, slot_term, slot_idf, slot_idf_f, ops, signals, k, slot_boost=None):
    """One query of the multi-field recall stage (orc_multi_signal_topk): `segments` = oracle Segments (one per field),
    `ops` = [(kind, field, chain, col, coeff)], `signals` = list of f64 columns.  Returns (docs, totals)."""
    L = _L()
    nf = len(segments)
    segs = (C.c_void_p * nf)(*[s.h for s in segments])
    cs = [np.ascontiguousarray(c, np.float32) for c in caches]
    carr = (C.c_void_p * nf)(*[c.ctypes.data for c in cs])
    sigs = [np.ascontiguousarray(x, np.float64) for x in signals]
    sarr = (C.c_void_p * max(len(sigs), 1))(*[x.ctypes.data for x in sigs])
    sf = np.ascontiguousarray(slot_field, np.uint8); keep = sf != 0xFF
    sf = np.ascontiguousarray(sf[keep]); st = np.ascontiguousarray(np.asarray(slot_term, np.uint32)[keep])
    i1 = np.ascontiguousarray(np.asarray(slot_idf, np.float32)[keep]); i2 = np.ascontiguousarray(np.asarray(slot_idf_f, np.float32)[keep])
    sb = None if slot_boost is None else np.ascontiguousarray(np.asarray(slot_boost, np.float64)[keep])
    o = np.array([[a, b, c_, d] for a, b, c_, d, _ in ops], np.uint32).reshape(-1, 4)
    oc = np.array([e for *_, e in ops], np.float64)
    docs = np.zeros(k, np.uint32); totals = np.zeros(k, np.float64); sc = C.c_uint64(0)
    n = L.orc_multi_signal_topk(nf, C.cast(segs, C.c_void_p), C.cast(carr, C.c_void_p), np.ascontiguousarray(k1s, np.float32),
                                np.ascontiguousarray(coefs, np.float32), sf.size, sf, st, i1, i2, None if sb is None else sb.ctypes.data, len(ops),
                                np.ascontiguousarray(o[:, 0]), np.ascontiguousarray(o[:, 1]), np.ascontiguousarray(o[:, 2]),
                                np.ascontiguousarray(o[:, 3]), oc, C.cast(sarr, C.c_void_p), k, docs, totals, C.byref(sc))
    return docs[:n], totals[:n]


def topn_f64(totals, docs, k):
    """The oracle's TopN<double> over (total, doc) pairs pushed in the given order.  Returns (docs, totals)."""
    t = np.ascontiguousarray(totals, np.float64); d = np.ascontiguousarray(docs, np.uint32)
    od = np.zeros(max(k, 1), np.uint32); ot = np.zeros(max(k, 1), np.float64)
    n = _L().orc_topn_f64(t, d, t.size, k, od, ot)
    return od[:n], ot[:n]


class Cursor:
    """TermScorer over SegmentPostings (term_scorer.rs)."""

    def __init__(self, seg, term, weight, cache):
        self.seg = seg
        self.L = seg.L
        self.h = self.L.orc_cursor_open(seg.h, term, float(weight), np.ascontiguousarray(cache, np.float32))

    def __getattr__(self, name):
        if name in ("doc", "tf", "advance", "last_doc_in_block", "score", "max_score", "block_max_score"):
            fn = getattr(self.L, f"orc_cursor_{name}")
            return lambda: fn(self.h)
        raise AttributeError(name)

    def seek(self, t):
        return self.L.orc_cursor_seek(self.h, t)

    def shallow_seek(self, t):
        self.L.orc_cursor_shallow_seek(self.h, t)

    def __del__(self):
        try:
            self.L.orc_cursor_free(self.h)
        except Exception:
            pass


# ---- TermInfoStore (tantivy/src/termdict/fst_termdict/term_info_store.rs) -------------------------------------------
def term_info_store_write(doc_freq, post_start, post_end, pos_start=None, pos_end=None):
    """TermInfoStoreWriter: bytes of the store for the given TermInfos (positions ranges default to empty)."""
    L = _L()
    df = np.ascontiguousarray(doc_freq, np.uint32); n = df.size
    ps = np.ascontiguousarray(post_start, np.uint64); pe = np.ascontiguousarray(post_end, np.uint64)
    qs = np.zeros(n, np.uint64) if pos_start is None else np.ascontiguousarray(pos_start, np.uint64)
    qe = np.zeros(n, np.uint64) if pos_end is None else np.ascontiguousarray(pos_end, np.uint64)
    ln = L.orc_tis_write(df, ps, pe, qs, qe, n, None)
    out = np.zeros(ln, np.uint8)
    L.orc_tis_write(df, ps, pe, qs, qe, n, out.ctypes.data)
    return out


def term_info_store_get(store, ord_):
    """TermInfoStore::get -> (doc_freq, postings_start, postings_end, positions_start, positions_end)."""
    L = _L()
    store = np.ascontiguousarray(store, np.uint8)
    df = C.c_uint32(); a, b, c, d = (C.c_uint64() for _ in range(4))
    L.orc_tis_get(store, store.size, int(ord_), C.byref(df), C.byref(a), C.byref(b), C.byref(c), C.byref(d))
    return df.value, a.value, b.value, c.value, d.value


def bitpack(vals, bits):
    L = _L()
    v = np.ascontiguousarray(vals, np.uint64); b = np.ascontiguousarray(bits, np.uint8)
    out = np.zeros(8 * v.size + 8, np.uint8)
    n = L.orc_bitpack(v, b, v.size, out)
    return out[:n]


def extract_bits(data, addr_bits, num_bits):
    d = np.ascontiguousarray(data, np.uint8)
    return int(_L().orc_extract_bits(d, d.size, int(addr_bits), int(num_bits)))


def numeric_scores(which, raw, now=None, region_counts=None, region_total=0, selected=None):
    """orc_numeric_scores: the value -> score transform of one numeric CoreSignal over a raw fast-field column
    (which: 0 identity f64, 1 score_rank, 2 IsHomepage, 3 HasAds, 4 inverse, 5 FetchTimeMs, 6 UpdateTimestamp, 7 LinkDensity, 8 Region)."""
    L = _L()
    fn = L.orc_numeric_scores
    fn.restype = None
    fn.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p, C.c_uint32, C.c_uint64, C.c_int64, C.c_void_p]
    u = f = b = None
    if which in (0, 7):
        f = np.ascontiguousarray(raw, np.float64); n = f.size
    elif which in (2, 3):
        b = np.ascontiguousarray(raw, np.uint8); n = b.size
    else:
        u = np.ascontiguousarray(raw, np.uint64); n = u.size
    rc = None if region_counts is None else np.array([-1 if c is None else int(c) for c in region_counts], np.int64)
    out = np.zeros(n, np.float64)
    fn(which, None if u is None else u.ctypes.data, None if f is None else f.ctypes.data, None if b is None else b.ctypes.data, n,
       -1 if now is None else int(now), None if rc is None else rc.ctypes.data, 0 if rc is None else rc.size, int(region_total),
       -1 if selected is None else int(selected), out.ctypes.data)
    return out
