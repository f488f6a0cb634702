"""CPU oracle (test infrastructure only -- see oracle/oracle_common.h).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this package.  It is a ctypes binding over oracle/liboracle.so (built by oracle/Makefile).
"""
from .pyoracle import *  # noqa: F401,F403
from .pyoracle_p2 import (Segment, Cursor, fieldnorm_to_id, id_to_fieldnorm, fieldnorms_to_ids,  # noqa: F401,E402
                         fieldnorm_table, tv_bm25_weight, stract_bm25_weight, term_info_store_write,
                         term_info_store_get, bitpack, extract_bits, multi_signal_topk, numeric_scores, topn_f64)
