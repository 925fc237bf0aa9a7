"""TEST INFRASTRUCTURE ONLY -- ctypes binding of the topic threshold checker (oracle/dsgd_oracle_topic_thresh.c).

`topic_thresh` answers for an Oracle of oracle/oracle.py (its CSR) and a row->topics CSR.  The library is oracle/oracle.py's
libdsgd_oracle.so.  Only tests/ and tools/ use it; the product package never does.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np

from . import oracle as _oracle
from .oracle import Oracle, _check, _p


def topic_thresh(orc: Oracle, topic_ptr, topic_id, n_topics: int, fbr: float = 0.0, W=None, idx=None, begin: int = 0,
                 n: Optional[int] = None, margins=None) -> Tuple[np.ndarray, np.ndarray]:
    """(thresholds, words) of dsgd_tune_topic_thresholds over the listed rows, or rows [begin, begin + n).  margins
    (optional, [T, n]): each topic's margins of the rows, tuned instead of the checker's own dots of W[T, dim]."""
    lib = _oracle.lib()
    lib.dsgd_oracle_topic_thresh.restype = C.c_int
    T = int(n_topics)
    if idx is not None:
        idx = orc._idx(idx)
        n = len(idx)
    elif n is None:
        n = orc.n_rows - begin
    tp = np.ascontiguousarray(topic_ptr, dtype=np.int64)
    ti = np.ascontiguousarray(topic_id, dtype=np.int32)
    assert tp.shape == (orc.n_rows + 1,) and ti.size == tp[-1]
    if margins is not None:
        margins = np.ascontiguousarray(margins, dtype=np.float64)
        assert margins.shape == (T, n)
        W = None
    else:
        W = np.ascontiguousarray(W, dtype=np.float64)
        assert W.shape == (T, orc.dim)
    thr = np.zeros(T, dtype=np.float64)
    words = np.zeros(8 * T, dtype=np.int64)
    _check(lib.dsgd_oracle_topic_thresh(C.byref(orc._csr), _p(W), C.c_int32(T), _p(tp), _p(ti), _p(idx),
                                        C.c_int64(begin), C.c_int64(n), _p(margins), C.c_double(fbr), _p(thr),
                                        _p(words)), "topic_thresh")
    return thr, words
