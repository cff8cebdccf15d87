"""Restatement of BTLE_CFG_OFFSET_SEARCH (include/btle_b200.h): the seven hypotheses' offsets and the merge of their records,
per (cfg, chunk).  The records of each hypothesis come from whatever decodes the call at that hypothesis's offsets (the
*_offset entry points on the GPU, the chain restatements on the CPU)."""
from __future__ import annotations

import numpy as np

from orc import REC_DTYPE

HYP_HZ = (0.0, -50e3, 50e3, -100e3, 100e3, -150e3, 150e3)   # BTLE_OFFSET_SEARCH_HZ, in merge order
REC_REJECTED, REC_OFFSET_SEARCH = 4, 128
WINDOW = 8                                                   # |n0 - r.n0| <= 8: the same packet (two symbols)
MAX_MERGED_RECS_PER_CHUNK = 123 + 6 * 51                     # BTLE_MAX_MERGED_RECS_PER_CHUNK


def hyp_offsets(f_c) -> list:
    """float32 [n] per hypothesis: f_c + delta_h, summed in float32 (f_c: a scalar or one value per capture)"""
    f = np.asarray(f_c, dtype=np.float32)
    return [(f + np.float32(d)).astype(np.float32) for d in HYP_HZ]


def ok(r) -> bool:
    """counted (not rejected, not raw) with a good CRC"""
    return (int(r["flags"]) & (REC_REJECTED | 1)) == 0 and int(r["crc_bad"]) == 0


def merge_chunk(hyps: list) -> list:
    """hyps[h]: hypothesis h's records of one (cfg, chunk), in n0 order -> the merged records of that (cfg, chunk)"""
    b = [r.copy() for r in hyps[0]]
    for h in range(1, len(HYP_HZ)):
        for r in hyps[h]:
            if not ok(r):
                continue
            near = [abs(int(x["n0"]) - int(r["n0"])) <= WINDOW for x in b]
            if any(n and ok(x) for n, x in zip(near, b)):
                continue
            b = [x for n, x in zip(near, b) if not n]
            r = r.copy()
            r["flags"] |= REC_OFFSET_SEARCH
            b.append(r)
            b.sort(key=lambda x: int(x["n0"]))
    return b


def merge(per_hyp: list, n_cfgs: int) -> np.ndarray:
    """per_hyp[h]: the records of the call at hypothesis h's offsets (stream = cfg index, in (cfg, chunk, n0) order) ->
    the records of the flagged call, in (cfg, chunk, n0) order"""
    out = []
    for j in range(n_cfgs):
        mine = [p[p["stream"] == j] for p in per_hyp]
        for k in sorted({int(c) for p in mine for c in p["chunk"]}):
            out += merge_chunk([p[p["chunk"] == k] for p in mine])
    return np.array(out, dtype=REC_DTYPE) if out else np.zeros(0, dtype=REC_DTYPE)
