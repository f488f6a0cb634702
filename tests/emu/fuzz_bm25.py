"""Corrupted-postings fuzz of the BM25 kernels (AND, OR, signal combine) on the CPU emulator; meant for the AddressSanitizer build:
    make -C tests/emu clean && make -C tests/emu SAN=1
    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python tests/emu/fuzz_bm25.py <seed> <trials>
Every corruption must end in a rejection at open, an SB200_EFORMAT at query time or a normal answer -- never in an
out-of-bounds access (this is how the missing doc-id range check before the fieldnorm / signal gathers was found)."""
import sys, ctypes as C, os, time
HERE = os.path.dirname(os.path.abspath(__file__)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE))); sys.path.insert(0, os.path.dirname(HERE))
import numpy as np
from stract_b200 import _lib
L = _lib.declare(C.CDLL(os.path.join(HERE, 'libsb200_emu.so'))); _lib._LIB = L
from stract_b200 import bm25
from stract_b200._lib import Sb200Error
from stract_b200.bm25 import MODE_AND, MODE_OR, SegmentReader, TopDocs, SignalComputer
rng = np.random.default_rng(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
max_doc = 20000
lens = np.maximum(1, rng.lognormal(4.0, 0.8, max_doc)).astype(np.uint32)
ids = bm25.fieldnorms_to_ids(lens)
dfs = [3, 127, 128, 300, 1000, 5000]
td = [np.sort(rng.choice(max_doc, df, replace=False)).astype(np.uint32) for df in dfs]
tt = [np.minimum(rng.geometric(0.6, df), 255).astype(np.uint32) for df in dfs]
good, infos = bm25.encode_postings(td, tt, ids, 60.0)
t0 = time.time(); n_rej = n_ok = n_qerr = 0
for trial in range(int(sys.argv[2]) if len(sys.argv) > 2 else 150):
    data = good.copy()
    for _ in range(int(rng.integers(1, 6))):
        i = int(rng.integers(0, data.size)); data[i] = rng.integers(0, 256)
    try:
        seg = SegmentReader(data, infos, ids)
    except Sb200Error:
        n_rej += 1; continue
    n_ok += 1
    for mode in (MODE_AND, MODE_OR):
        q = np.array([[5, 4], [3, 5], [2, 1], [5, 0]], np.uint32)
        try:
            TopDocs.with_limit(50).search_batch(seg, q, mode)
        except Sb200Error:
            n_qerr += 1
    try:
        SignalComputer(seg, None, (), coeff_text=1.0).top_docs_batch(np.array([[5, 4, 3]], np.uint32), 20)
    except Sb200Error:
        n_qerr += 1
    seg.close()
print("fuzz done: rejected at open", n_rej, "opened", n_ok, "query errors", n_qerr, "in", round(time.time() - t0), "s")
