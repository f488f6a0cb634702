"""The native threaded phrase oracle (tests/phrase_oracle_mt.cpp: the CPU baseline and full-size parity reference of
tools/phrase_bench.py) against the Python oracle, which test_oracle_phrase.py pins on the reference's tests.  No GPU."""
import numpy as np
import pytest

import phrase_oracle as O
from phrase_fixtures import index_to_csr, native_batch, random_index, random_rows


@pytest.mark.parametrize("scoring", [True, False])
def test_native_oracle_equals_python_oracle(scoring):
    from stract_b200.bm25 import NO_TERM, id_to_fieldnorm
    index, rng = random_index(3, 500, long_doc=300)
    csr = index_to_csr(index)
    n = index["fieldnorm_ids"].size
    avg = np.float32(np.float32(index["total_num_tokens"]) / np.float32(n))
    cache = O.tf_cache(avg, [id_to_fieldnorm(i) for i in range(256)])
    for width in (2, 3, 6):
        rows, offs = random_rows(rng, len(index["terms"]) - 2, 12, width)
        for slop in (0, 1, 3, 300):
            slops = np.full(12, slop, np.uint32)
            ws, want = [], []
            for q in range(12):
                real = [j for j in range(width) if rows[q, j] != NO_TERM]
                terms = [None if rows[q, j] == 0xFFFFFFFE else int(rows[q, j]) for j in real]
                w = O.bm25_weight_for_terms([0 if t is None else len(index["terms"][t]["docs"]) for t in terms], n)
                ws.append(w)
                want.append(O.phrase_search(index, terms, [int(offs[q, j]) for j in real], slop, scoring, w, cache, 50))
            d, s, c = native_batch(csr, rows, offs, slops, ws, cache, scoring, 50, threads=4)
            for q, hits in enumerate(want):
                assert int(c[q]) == len(hits), (width, slop, q)
                assert d[q, :c[q]].tolist() == [h[1] for h in hits]
                assert np.array_equal(s[q, :c[q]].view(np.uint32), np.array([h[0] for h in hits], np.float32).view(np.uint32))
