"""ctypes binding of the C-ABI (include/btle_b200.h -> btle_b200/libbtle_b200.so).

There is no CPU fallback: if the CUDA library is missing or no CUDA device is usable this module
raises.  Nothing here imports the test oracle."""
from __future__ import annotations

import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BTLE_B200_LIB") or os.path.join(_HERE, "libbtle_b200.so")   # env override: A/B builds

BTLE_OK, BTLE_EINVAL, BTLE_ENODEV, BTLE_ENOMEM, BTLE_ECUDA, BTLE_EOVERFLOW = 0, -1, -2, -3, -4, -5

# btle_pkt_rec, 64 bytes
REC_DTYPE = np.dtype([
    ("stream", "<i4"), ("chunk", "<i4"), ("n0", "<i4"),
    ("channel", "u1"), ("n_bytes", "u1"), ("crc_bad", "u1"), ("flags", "u1"),
    ("access_addr", "<u4"), ("mag_sum", "<u2"), ("bytes", "u1", 42),
])
# btle_stream_cfg, 24 bytes
CFG_DTYPE = np.dtype([("channel", "<i4"), ("access_addr", "<u4"), ("access_mask", "<u4"), ("crc_init", "<u4"),
                      ("raw", "<i4"), ("rssi", "<i4")])
# btle_model_rx_rec, 80 bytes
MODEL_REC_DTYPE = np.dtype([("start", "<i4"), ("n_pdu_bits", "<u2"), ("crc_ok", "u1"), ("phase", "u1"), ("payload_len", "u1"),
                            ("found", "u1"), ("pdu", "u1", 70)])
# btle_synth_cfg (32 bytes) / btle_synth_truth (64 bytes)
SYNTH_CFG_DTYPE = np.dtype([("seed", "<u8"), ("slot_samples", "<i4"), ("amplitude", "<i4"), ("corrupt_every", "<i4"),
                            ("straddle_every", "<i4"), ("noise", "<i4"), ("reserved", "<i4")])
SYNTH_TRUTH_DTYPE = np.dtype([("start_sample", "<i8"), ("stream", "<i4"), ("slot", "<i4"), ("n_air_bytes", "u1"), ("corrupt", "u1"),
                              ("straddle", "u1"), ("pdu_len", "u1"), ("pdu", "u1", 44)])
assert SYNTH_CFG_DTYPE.itemsize == 32 and SYNTH_TRUTH_DTYPE.itemsize == 64
DIR_DTYPE = np.dtype([("base", "<u4"), ("count", "<u4")])      # btle_unit_dir
BER_CFG_DTYPE = np.dtype([("seed", "<u8"), ("snr_db", "<f4"), ("ppm", "<f4"), ("channel", "<i4"), ("crc_init", "<u4"), ("access_addr", "<u4"),
                          ("reserved", "<u4")])
BER_RESULT_DTYPE = np.dtype([("packets", "<u8"), ("pkt_err", "<u8"), ("bit_err", "<u8"), ("bit_total", "<u8"), ("aa_miss", "<u8"), ("seconds", "<f8")])
assert BER_CFG_DTYPE.itemsize == 32 and BER_RESULT_DTYPE.itemsize == 48
# btle_rx_ber_cfg (48 bytes), btle_rx_ber_truth (64 bytes), btle_rx_ber_result (88 bytes): error rates of the 4-Msps receiver
RX_BER_CFG_DTYPE = np.dtype([("seed", "<u8"), ("snr_db", "<f4"), ("ppm", "<f4"), ("cfo_hz", "<f4"), ("amplitude", "<i4"), ("slot_samples", "<i4"),
                             ("channel", "<i4"), ("access_addr", "<u4"), ("crc_init", "<u4"), ("flags", "<u4"), ("reserved", "<u4")])
RX_BER_TRUTH_DTYPE = np.dtype([("aa_sample", "<i8"), ("offset", "<i4"), ("clipped", "<u4"), ("n_bytes", "u1"), ("delta4", "u1"), ("pdu", "u1", 39),
                               ("reserved", "u1", 7)])
RX_BER_COUNTERS = ("packets", "pkt_err", "bit_err", "bit_total", "aa_miss", "len_reject", "crc_ok_wrong", "extra_recs", "extra_crc_ok", "clipped")
RX_BER_RESULT_DTYPE = np.dtype([(k, "<u8") for k in RX_BER_COUNTERS] + [("seconds", "<f8")])
assert RX_BER_CFG_DTYPE.itemsize == 48 and RX_BER_TRUTH_DTYPE.itemsize == 64 and RX_BER_RESULT_DTYPE.itemsize == 88
RX_BER_MAX_SLOT, RX_BER_MAX_UNITS = 12000, 12272       # BTLE_RX_BER_MAX_SLOT, BTLE_RX_BER_MAX_UNITS
SPS8_REC_DTYPE = np.dtype([("sample", "<i8"), ("window", "<i8"), ("rx", MODEL_REC_DTYPE)])     # btle_sps8_rec
# btle_conn_cand, 32 bytes: an empty-PDU candidate of connection discovery
CAND_DTYPE = np.dtype([("sample", "<i8"), ("stream", "<i4"), ("access_addr", "<u4"), ("crc_init", "<u4"), ("channel", "u1"),
                       ("header", "u1", 2), ("reserved", "u1", 9)])
assert CAND_DTYPE.itemsize == 32
# btle_coded_rec, 304 bytes: one LE Coded PHY packet (btle_b200_rx_coded)
CODED_MAX_BYTES = 260
CODED_REC_DTYPE = np.dtype([("sample", "<i8"), ("stream", "<i4"), ("access_addr", "<u4"), ("channel", "u1"), ("s", "u1"), ("ci", "u1"),
                            ("crc_bad", "u1"), ("flags", "u1"), ("reserved0", "u1"), ("n_bytes", "<u2"), ("dist", "<i4"), ("metric", "<i4"),
                            ("mag_sum", "<u4"), ("bytes", "u1", CODED_MAX_BYTES), ("reserved", "u1", 8)])
assert CODED_REC_DTYPE.itemsize == 304
CODED_MAX_DIST = 96                           # BTLE_CODED_MAX_DIST
# btle_coded_cand, 32 bytes: an empty coded PDU candidate of coded connection discovery (first 23 bytes as CAND_DTYPE)
CODED_CAND_DTYPE = np.dtype([("sample", "<i8"), ("stream", "<i4"), ("access_addr", "<u4"), ("crc_init", "<u4"), ("channel", "u1"),
                             ("header", "u1", 2), ("s", "u1"), ("dist", "<i2"), ("shift", "i1"), ("reserved", "u1"), ("metric", "<i4")])
assert CODED_CAND_DTYPE.itemsize == 32
CODED_CI_RESERVED, CODED_TRUNCATED = 1, 2     # btle_coded_rec.flags bits
assert REC_DTYPE.itemsize == 64 and CFG_DTYPE.itemsize == 24 and MODEL_REC_DTYPE.itemsize == 80 and SPS8_REC_DTYPE.itemsize == 96

EXPORTS = [
    "btle_b200_create", "btle_b200_destroy", "btle_b200_bind_host_numa", "btle_b200_last_error", "btle_b200_strerror", "btle_b200_version",
    "btle_b200_rx_batch", "btle_b200_rx", "btle_b200_rx_device", "btle_b200_rx_device_dir", "btle_b200_rx_units",
    "btle_b200_gather_ordered", "btle_b200_sort_records", "btle_b200_last_launches",
    "btle_b200_search_unique_bits", "btle_b200_demod_byte", "btle_b200_scramble_byte", "btle_b200_crc24_byte",
    "btle_b200_crc_init_reorder", "btle_b200_parse_adv_pdu_header_byte", "btle_b200_parse_ll_pdu_header_byte",
    "btle_b200_dbits", "btle_b200_gfsk_demod_i16", "btle_b200_search_bit_sequence", "btle_b200_crc24_bits",
    "btle_b200_scramble_bits", "btle_b200_model_rx_batch_device", "btle_b200_model_rx_batch",
    "btle_b200_tx_modulate_device", "btle_b200_rx_iq16", "btle_b200_synth_streams_device", "btle_b200_rx_sps8", "btle_b200_sps8_hits_device", "btle_b200_ber_run",
    "btle_b200_ber_synth_device", "btle_b200_rx_ber_run", "btle_b200_rx_ber_synth_device", "btle_b200_rx_ber_score_device",
    "btle_b200_stream_open", "btle_b200_stream_push", "btle_b200_stream_acquire", "btle_b200_stream_commit", "btle_b200_stream_finish",
    "btle_b200_stream_close", "btle_b200_stream_set_cfg",
    "btle_b200_streams_open", "btle_b200_streams_acquire", "btle_b200_streams_commit", "btle_b200_streams_set_cfg",
    "btle_b200_streams_finish", "btle_b200_streams_close", "btle_b200_parse_adv_pdu_payload_byte", "btle_b200_parse_ll_pdu_payload_byte",
    "btle_b200_receiver_controller", "btle_b200_receiver_status", "btle_b200_note_packet", "btle_b200_set_hop_hooks", "btle_b200_hop_reset",
    "btle_b200_get_freq_by_channel_number", "btle_b200_chm_is_full_map", "btle_b200_discover", "btle_b200_discover_device",
    "btle_b200_rx_multi", "btle_b200_rx_multi_units", "btle_b200_rx_multi_device_dir",
    "btle_b200_streams_add_cfg", "btle_b200_streams_remove_cfg", "btle_b200_streams_resident", "btle_b200_streams_set_discover",
    "btle_b200_streams_take_cands", "btle_b200_rx_batch_offset", "btle_b200_rx_device_dir_offset", "btle_b200_rx_multi_offset",
    "btle_b200_rx_multi_device_dir_offset", "btle_b200_rec_offset_device", "btle_b200_rec_offset",
    "btle_b200_streams_set_offset", "btle_b200_stream_set_offset", "btle_b200_rx_coded", "btle_b200_rx_coded_device",
    "btle_b200_rx_coded_multi", "btle_b200_rx_coded_multi_device", "btle_b200_discover_coded", "btle_b200_discover_coded_device",
]
MAX_CFGS_PER_CAPTURE = 8       # BTLE_MAX_CFGS_PER_CAPTURE
CFG_RSSI, CFG_REPORT_REJECTED, CFG_RECOVER = 1, 2, 4      # btle_stream_cfg.rssi flag bits (BTLE_CFG_*)
CFG_SYMBOL_SPACED = 16       # BTLE_CFG_SYMBOL_SPACED: symbol-spaced discriminator (one mode per launch / session)
CFG_CENTRE_HITS = 64         # BTLE_CFG_CENTRE_HITS: each hit moved to the centre of its run of matching sample phases (per cfg)
CFG_CORRECT = 256            # BTLE_CFG_CORRECT: one-bit and adjacent-pair errors of CRC-failed packets corrected (per cfg)
CFG_LOWPASS = 512            # BTLE_CFG_LOWPASS: [1, 2, 1] low-pass in front of the symbol-spaced bits (with CFG_SYMBOL_SPACED, one mode per launch)
MAX_OFFSET_HZ = 500000       # BTLE_MAX_OFFSET_HZ: largest |offset_hz| of the carrier-offset correction
CFG_OFFSET_SEARCH = 1024     # BTLE_CFG_OFFSET_SEARCH: seven carrier-offset hypotheses per capture, merged per packet (one mode per launch)
OFFSET_SEARCH_HZ = (0.0, -50e3, 50e3, -100e3, 100e3, -150e3, 150e3)   # BTLE_OFFSET_SEARCH_HZ: the hypotheses, in merge order
MAX_MERGED_RECS_PER_CHUNK = 429                           # BTLE_MAX_MERGED_RECS_PER_CHUNK = 123 + 6 * 51
REC_REJECTED, REC_RECOVERED = 4, 8                        # btle_pkt_rec.flags bits; a recovered record's alternative q is flags >> 4 & 3
REC_CORRECTED = 64                                        # btle_pkt_rec.flags bit: bytes corrected by the CRC syndrome
REC_OFFSET_SEARCH = 128                                   # btle_pkt_rec.flags bit: found by offset hypothesis 1..6 (CFG_OFFSET_SEARCH)


class BtleError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"btle_b200 error {code}: {msg}")
        self.code = code


_lib = None


def load():
    """Load libbtle_b200.so (built in-tree by __graft_entry__.build()).  Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BtleError(BTLE_ENODEV, f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
    L = ctypes.CDLL(LIB_PATH)
    vp, sz, i32, u32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint32
    L.btle_b200_create.argtypes = [ctypes.POINTER(vp), i32]
    L.btle_b200_bind_host_numa.argtypes = [i32, ctypes.POINTER(ctypes.c_int)]
    L.btle_b200_destroy.argtypes = [vp]
    L.btle_b200_destroy.restype = None
    L.btle_b200_last_error.argtypes = [vp]
    L.btle_b200_last_error.restype = ctypes.c_char_p
    L.btle_b200_strerror.argtypes = [i32]
    L.btle_b200_strerror.restype = ctypes.c_char_p
    L.btle_b200_version.restype = u32
    L.btle_b200_rx_batch.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_rx.argtypes = [vp, vp, sz, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_rx_device.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, vp]
    L.btle_b200_rx_device_dir.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, vp, sz, vp]
    L.btle_b200_rx_units.argtypes = [vp, sz, sz]
    L.btle_b200_rx_units.restype = sz
    L.btle_b200_gather_ordered.argtypes = [vp, sz, vp, sz, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_sort_records.argtypes = [vp, sz]
    L.btle_b200_sort_records.restype = None
    L.btle_b200_last_launches.argtypes = [vp]
    L.btle_b200_search_unique_bits.argtypes = [vp, vp, i32, vp, vp, i32]
    L.btle_b200_demod_byte.argtypes = [vp, vp, i32, vp]
    L.btle_b200_scramble_byte.argtypes = [vp, vp, i32, i32, i32, vp]
    L.btle_b200_crc24_byte.argtypes = [vp, vp, i32, u32, ctypes.POINTER(u32)]
    L.btle_b200_crc_init_reorder.argtypes = [u32]
    L.btle_b200_crc_init_reorder.restype = u32
    ip = ctypes.POINTER(ctypes.c_int)
    L.btle_b200_parse_adv_pdu_header_byte.argtypes = [vp, ip, ip, ip, ip]
    L.btle_b200_parse_adv_pdu_header_byte.restype = None
    L.btle_b200_parse_ll_pdu_header_byte.argtypes = [vp, ip, ip, ip, ip, ip]
    L.btle_b200_parse_ll_pdu_header_byte.restype = None
    L.btle_b200_dbits.argtypes = [vp, vp, sz, vp]
    L.btle_b200_gfsk_demod_i16.argtypes = [vp, vp, vp, sz, vp, vp]
    L.btle_b200_search_bit_sequence.argtypes = [vp, vp, sz, vp, sz]
    L.btle_b200_search_bit_sequence.restype = ctypes.c_long
    L.btle_b200_crc24_bits.argtypes = [vp, vp, sz, vp, vp]
    L.btle_b200_scramble_bits.argtypes = [vp, vp, sz, i32, vp]
    L.btle_b200_model_rx_batch_device.argtypes = [vp, vp, vp, sz, sz, i32, i32, u32, u32, vp, vp]
    L.btle_b200_model_rx_batch.argtypes = [vp, vp, vp, sz, sz, i32, i32, u32, u32, vp]
    L.btle_b200_tx_modulate_device.argtypes = [vp, vp, vp, sz, sz, i32, vp, vp, vp]
    L.btle_b200_rx_iq16.argtypes = [vp, vp, sz, i32, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_ber_run.argtypes = [vp, vp, sz, vp]
    L.btle_b200_ber_synth_device.argtypes = [vp, vp, ctypes.c_uint64, sz, vp, vp, vp, vp]
    L.btle_b200_rx_ber_run.argtypes = [vp, vp, sz, vp]
    L.btle_b200_rx_ber_synth_device.argtypes = [vp, vp, ctypes.c_uint64, sz, vp, vp, vp]
    L.btle_b200_rx_ber_score_device.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, vp]
    L.btle_b200_sps8_hits_device.argtypes = [vp, vp, sz, u32, vp, sz, vp, vp]
    L.btle_b200_rx_sps8.argtypes = [vp, vp, sz, i32, u32, u32, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_synth_streams_device.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, sz, ctypes.POINTER(sz), vp]
    L.btle_b200_stream_open.argtypes = [vp, vp, sz, ctypes.POINTER(vp)]
    L.btle_b200_stream_acquire.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(sz)]
    L.btle_b200_stream_commit.argtypes = [vp, sz, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_stream_push.argtypes = [vp, vp, sz, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_stream_set_cfg.argtypes = [vp, vp]
    L.btle_b200_stream_finish.argtypes = [vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_stream_close.argtypes = [vp]
    L.btle_b200_stream_close.restype = None
    L.btle_b200_streams_open.argtypes = [vp, vp, sz, sz, ctypes.POINTER(vp)]
    L.btle_b200_streams_acquire.argtypes = [vp, sz, ctypes.POINTER(vp), ctypes.POINTER(sz)]
    L.btle_b200_streams_commit.argtypes = [vp, sz, sz, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_streams_set_cfg.argtypes = [vp, sz, vp]
    L.btle_b200_streams_finish.argtypes = [vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_streams_close.argtypes = [vp]
    L.btle_b200_streams_close.restype = None
    L.btle_b200_discover.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_discover_device.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, vp]
    L.btle_b200_rx_multi.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_rx_multi_units.argtypes = [vp, sz, vp, sz, sz]
    L.btle_b200_rx_multi_units.restype = sz
    L.btle_b200_rx_multi_device_dir.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, sz, vp, vp, sz, vp]
    i64p = ctypes.POINTER(ctypes.c_int64)
    L.btle_b200_streams_add_cfg.argtypes = [vp, sz, vp, ctypes.c_int64, ctypes.POINTER(sz)]
    L.btle_b200_streams_remove_cfg.argtypes = [vp, sz, i64p]
    L.btle_b200_streams_resident.argtypes = [vp, i64p]
    L.btle_b200_streams_set_discover.argtypes = [vp, vp]
    L.btle_b200_streams_take_cands.argtypes = [vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_rx_batch_offset.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_rx_device_dir_offset.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, sz, vp, vp, sz, vp]
    L.btle_b200_rx_multi_offset.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_rx_multi_device_dir_offset.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, vp, sz, vp, vp, sz, vp]
    L.btle_b200_rec_offset_device.argtypes = [vp, vp, sz, sz, vp, sz, vp, vp]
    L.btle_b200_rec_offset.argtypes = [vp, vp, sz, sz, sz, vp, sz, vp]
    L.btle_b200_streams_set_offset.argtypes = [vp, sz, ctypes.c_float]
    L.btle_b200_stream_set_offset.argtypes = [vp, ctypes.c_float]
    L.btle_b200_rx_coded.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_rx_coded_device.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, sz, vp, vp]
    L.btle_b200_rx_coded_multi.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_rx_coded_multi_device.argtypes = [vp, vp, sz, sz, sz, vp, vp, sz, vp, vp, sz, vp, vp]
    L.btle_b200_discover_coded.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, sz, ctypes.POINTER(sz)]
    L.btle_b200_discover_coded_device.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, sz, vp, vp]
    _lib = L
    return L


def bind_host_numa(device: int) -> int:
    """Bind the calling thread (CPU affinity + preferred memory node) to the NUMA node of CUDA device `device`
    (btle_b200_bind_host_numa).  Returns the node or -1."""
    node = ctypes.c_int(-1)
    load().btle_b200_bind_host_numa(int(device), ctypes.byref(node))
    return node.value
