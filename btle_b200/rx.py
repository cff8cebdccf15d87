"""Python face of the receive path: thin object over the C-ABI context.

`BtleRx.rx()` / `rx_batch()` take host int8 IQ (numpy) and return packet records
(numpy structured array, `REC_DTYPE`) in the order the reference's receiver() emits them.
`rx_device()` works on CUDA tensors already resident in HBM (torch is only used for the
device memory and the stream)."""
from __future__ import annotations

import ctypes
from functools import partial

import numpy as np

from . import _native
from ._native import BTLE_EOVERFLOW, BtleError, CAND_DTYPE, CFG_DTYPE, DIR_DTYPE, REC_DTYPE

DEFAULT_ACCESS_ADDR = 0x8E89BED6     # btle_rx.c:231
DEFAULT_CRC_INIT = 0x555555          # btle_rx.c:232
DEFAULT_CHANNEL = 37                 # btle_rx.c:230


def make_cfgs(n_streams=1, channel=DEFAULT_CHANNEL, access_addr=DEFAULT_ACCESS_ADDR, access_mask=0xFFFFFFFF,
              crc_init=DEFAULT_CRC_INIT, raw=0, rssi=0, recover=0) -> np.ndarray:
    """btle_stream_cfg array; every argument may be a scalar or a per-stream sequence.  rssi holds the BTLE_CFG_* flag
    bits; recover (true) adds BTLE_CFG_RECOVER: counted packets that fail the CRC are demodulated again
    (include/btle_b200.h)."""
    c = np.zeros(n_streams, dtype=CFG_DTYPE)
    c["channel"], c["access_addr"], c["access_mask"] = channel, access_addr, access_mask
    c["crc_init"], c["raw"], c["rssi"] = crc_init, raw, rssi
    c["rssi"] |= np.where(np.asarray(recover) != 0, _native.CFG_RECOVER, 0).astype(np.int32)
    return c


def _with_fields(c: np.ndarray, cfg: dict) -> np.ndarray:
    """c (a btle_stream_cfg array) with the given make_cfgs fields changed; recover sets or clears BTLE_CFG_RECOVER"""
    for k, v in cfg.items():
        if k == "recover":
            c["rssi"] = (c["rssi"] & ~_native.CFG_RECOVER) | (_native.CFG_RECOVER if v else 0)
        else:
            c[k] = v
    return c


def _offsets(offset_hz, n: int):
    """float32 [n] of a scalar or per-capture offset, or None (no correction: the default kernels)"""
    if offset_hz is None:
        return None
    return np.ascontiguousarray(np.broadcast_to(np.asarray(offset_hz, dtype=np.float32), (n,)))


def _ptr(a):
    """a's data pointer, or None (NULL) for None"""
    return None if a is None else a.ctypes.data


class BtleRx:
    def __init__(self, device: int = 0):
        self._L = _native.load()
        h = ctypes.c_void_p()
        rc = self._L.btle_b200_create(ctypes.byref(h), int(device))
        if rc != 0:
            raise BtleError(rc, self._L.btle_b200_strerror(rc).decode())
        self._h = h
        self.device = int(device)

    def close(self):
        if getattr(self, "_h", None):
            self._L.btle_b200_destroy(self._h)
            self._h = None

    __del__ = close

    def _check(self, rc):
        if rc != 0:
            raise BtleError(rc, self._L.btle_b200_last_error(self._h).decode() or self._L.btle_b200_strerror(rc).decode())

    @property
    def last_launches(self) -> int:
        return self._L.btle_b200_last_launches(self._h)

    def _grow_once(self, call, dtype, cap: int, grow: bool = True) -> np.ndarray:
        """call(out, cap, n_out) into `cap` records of `dtype`; on BTLE_EOVERFLOW, when `grow`, once more with the exact
        count it reported."""
        while True:
            out = np.empty(cap, dtype=dtype)
            n_out = ctypes.c_size_t(0)
            rc = call(out.ctypes.data, cap, ctypes.byref(n_out))
            if rc == BTLE_EOVERFLOW and grow:
                cap, grow = n_out.value, False
                continue
            self._check(rc)
            return out[:n_out.value]

    def _drain(self, finish, h, buf: np.ndarray) -> np.ndarray:
        """finish(h, buf, size, n_out) until it stops returning BTLE_EOVERFLOW: every record it hands out."""
        out = []
        while True:
            n = ctypes.c_size_t(0)
            rc = finish(h, buf.ctypes.data, buf.size, ctypes.byref(n))
            out.append(buf[:n.value].copy())
            if rc != BTLE_EOVERFLOW:
                self._check(rc)
                return np.concatenate(out)

    # ---- host buffers -------------------------------------------------------------------
    def rx_batch(self, iq: np.ndarray, cfgs: np.ndarray, cap: int | None = None, offset_hz=None) -> np.ndarray:
        """iq: int8 [n_streams, n_int8] (C-contiguous) or [n_int8]; cfgs: CFG_DTYPE [n_streams].  offset_hz (a scalar or one
        per capture, Hz, received minus nominal carrier): carrier-offset correction (btle_b200_rx_batch_offset)."""
        iq = np.ascontiguousarray(iq, dtype=np.int8)
        if iq.ndim == 1:
            iq = iq[None, :]
        ns, n = iq.shape
        cfgs = np.ascontiguousarray(cfgs, dtype=CFG_DTYPE)
        assert cfgs.shape == (ns,)
        off = _offsets(offset_hz, ns)
        # default capacity: typical worst case; grown once on BTLE_EOVERFLOW to the exact count, which is at most
        # BTLE_MAX_PKTS_PER_CHUNK (51) records per chunk, or BTLE_MAX_RECS_PER_CHUNK (123) with BTLE_CFG_REPORT_REJECTED
        call = partial(self._L.btle_b200_rx_batch_offset, self._h, iq.ctypes.data, ns, n, n, cfgs.ctypes.data, _ptr(off))
        return self._grow_once(call, REC_DTYPE, ns * (n // 16384) * 34 + 16 if cap is None else cap, grow=cap is None)

    def rx_multi(self, iq: np.ndarray, cfgs: np.ndarray, capture, cap: int | None = None, offset_hz=None) -> np.ndarray:
        """Several cfgs per capture in one read of the IQ (btle_b200_rx_multi): iq int8 [n_captures, n_int8] (or [n_int8]);
        cfgs CFG_DTYPE [n_cfgs]; capture[j] = the capture cfg j decodes (non-decreasing, at most MAX_CFGS_PER_CAPTURE
        per capture).  Returns what rx_batch() returns on iq[capture] with cfgs: records with stream = cfg index, in
        (cfg, chunk, n0) order.  offset_hz: a scalar or one per capture (carrier-offset correction)."""
        iq = np.ascontiguousarray(iq, dtype=np.int8)
        if iq.ndim == 1:
            iq = iq[None, :]
        ns, n = iq.shape
        cfgs = np.ascontiguousarray(cfgs, dtype=CFG_DTYPE).reshape(-1)
        cc = np.ascontiguousarray(capture, dtype=np.int32).reshape(-1)
        assert cc.shape == cfgs.shape
        off = _offsets(offset_hz, ns)
        call = partial(self._L.btle_b200_rx_multi_offset, self._h, iq.ctypes.data, ns, n, n, cfgs.ctypes.data, cc.ctypes.data, cfgs.size,
                       _ptr(off))
        return self._grow_once(call, REC_DTYPE, cfgs.size * (n // 16384) * 34 + 16 if cap is None else cap, grow=cap is None)

    def multi_units(self, n_captures: int, capture, n_int8: int) -> int:
        """Number of unit-directory entries an rx_multi launch over this shape writes (btle_b200_rx_multi_units)."""
        cc = np.ascontiguousarray(capture, dtype=np.int32).reshape(-1)
        return int(self._L.btle_b200_rx_multi_units(self._h, n_captures, cc.ctypes.data, cc.size, n_int8))

    def rx_multi_device_dir(self, d_iq, cfgs: np.ndarray, capture, d_out, d_count, d_dir, stream_ptr: int = 0, offset_hz=None):
        """rx_multi on device-resident captures, buffers as rx_device_dir (d_count may be None); d_dir holds at least
        multi_units(...) * 8 bytes.  gather_ordered() of the launch gives rx_multi()'s result.  offset_hz as rx_multi."""
        ns, n = d_iq.shape
        cfgs = np.ascontiguousarray(cfgs, dtype=CFG_DTYPE).reshape(-1)
        cc = np.ascontiguousarray(capture, dtype=np.int32).reshape(-1)
        assert d_iq.stride(1) == 1 and cc.shape == cfgs.shape
        cap = d_out.numel() * d_out.element_size() // 64
        dir_cap = d_dir.numel() * d_dir.element_size() // 8
        off = _offsets(offset_hz, ns)
        self._check(self._L.btle_b200_rx_multi_device_dir_offset(
            self._h, d_iq.data_ptr(), ns, d_iq.stride(0), n, cfgs.ctypes.data, cc.ctypes.data, cfgs.size, _ptr(off), d_out.data_ptr(), cap,
            d_count.data_ptr() if d_count is not None else None, d_dir.data_ptr(), dir_cap, ctypes.c_void_p(stream_ptr)))

    def rx(self, iq: np.ndarray, offset_hz=None, **cfg) -> np.ndarray:
        return self.rx_batch(np.asarray(iq).reshape(1, -1), make_cfgs(1, **cfg), offset_hz=offset_hz)

    # ---- carrier offset -------------------------------------------------------------------
    def rec_offsets(self, iq: np.ndarray, recs: np.ndarray) -> np.ndarray:
        """float32 [len(recs)]: the carrier-offset estimate of each record in Hz (btle_b200_rec_offset; definition in
        include/btle_b200.h).  iq as rx_batch's; a record's `stream` is its capture."""
        iq = np.ascontiguousarray(iq, dtype=np.int8)
        if iq.ndim == 1:
            iq = iq[None, :]
        ns, n = iq.shape
        recs = np.ascontiguousarray(recs, dtype=REC_DTYPE)
        hz = np.zeros(recs.size, dtype=np.float32)
        self._check(self._L.btle_b200_rec_offset(self._h, iq.ctypes.data, ns, n, n, recs.ctypes.data, recs.size, hz.ctypes.data))
        return hz

    def estimate_offset(self, iq: np.ndarray, **cfg):
        """Carrier offset of one capture in Hz: decoded without correction, the median of the per-record estimates
        (btle_b200_rec_offset_device) over the counted records with a good CRC; None when there is none.  The capture is
        copied to the device once and both passes read that copy.  Pass the result back as rx(..., offset_hz=)."""
        import torch
        iq = np.ascontiguousarray(np.asarray(iq, dtype=np.int8).reshape(1, -1))
        n = iq.shape[1]
        dev = torch.device("cuda", self.device)
        st = torch.cuda.current_stream(dev)
        d_iq = torch.from_numpy(np.pad(iq, ((0, 0), (0, -n % 16)))).to(dev)[:, :n]
        cap = (n // 16384) * 123 + 16                                   # BTLE_MAX_RECS_PER_CHUNK per chunk: never an overflow
        d_out = torch.empty(cap * 64, dtype=torch.uint8, device=dev)
        d_dir = torch.empty(max(self.units(1, n), 1) * 8, dtype=torch.uint8, device=dev)
        self.rx_device_dir(d_iq, make_cfgs(1, **cfg), d_out, None, d_dir, st.cuda_stream)
        st.synchronize()
        recs = self.gather_ordered(d_out.cpu().numpy().view(REC_DTYPE), d_dir.cpu().numpy().view(DIR_DTYPE))
        ok = np.ascontiguousarray(recs[(recs["crc_bad"] == 0) & ((recs["flags"] & (1 | _native.REC_REJECTED)) == 0)])
        if ok.size == 0:
            return None
        d_ok = torch.from_numpy(ok.view(np.uint8).copy()).to(dev)
        d_hz = torch.empty(ok.size, dtype=torch.float32, device=dev)
        self.rec_offsets_device(d_iq, d_ok, ok.size, d_hz, st.cuda_stream)
        st.synchronize()
        return float(np.median(d_hz.cpu().numpy()))

    def rx_iq16(self, iq16: np.ndarray, shift: int = 4, **cfg) -> np.ndarray:
        """int16 interleaved IQ (bladeRF SC16Q11: shift 4, btle_rx.c:307-308) -> records."""
        iq16 = np.ascontiguousarray(iq16, dtype=np.int16)
        cfgs = make_cfgs(1, **cfg)
        return self._grow_once(partial(self._L.btle_b200_rx_iq16, self._h, iq16.ctypes.data, iq16.size, shift, cfgs.ctypes.data), REC_DTYPE,
                               (iq16.size // 16384) * 34 + 16)

    def rx_sps8(self, iq16: np.ndarray, channel=DEFAULT_CHANNEL, crc_init=DEFAULT_CRC_INIT, access_addr=DEFAULT_ACCESS_ADDR) -> np.ndarray:
        """Interleaved int16 I,Q at 8 samples per symbol (a `btle_ll -q` .bin capture) -> SPS8_REC_DTYPE array: the Python
        model's receiver (8 phases, first CRC-ok phase wins) on every packet the GPU finds in the capture."""
        from ._native import SPS8_REC_DTYPE
        iq16 = np.ascontiguousarray(iq16, dtype=np.int16).reshape(-1)
        n = iq16.size // 2
        cap = n // 576 + 16
        out = np.zeros(cap, dtype=SPS8_REC_DTYPE)
        n_out = ctypes.c_size_t(0)
        self._check(self._L.btle_b200_rx_sps8(self._h, iq16.ctypes.data, n, int(channel), int(crc_init), int(access_addr), out.ctypes.data, cap,
                                              ctypes.byref(n_out)))
        return out[:n_out.value]

    def discover(self, iq: np.ndarray, channels, cap: int | None = None) -> np.ndarray:
        """Empty-PDU candidates of connection discovery (btle_b200_discover): iq int8 [n_streams, n_int8] (or [n_int8]) of
        data-channel captures, channels[s] in 0..36 the channel of capture s.  Returns CAND_DTYPE records sorted by
        (stream, sample); `cap` defaults to a typical worst case and is grown once to the exact count on overflow."""
        iq = np.ascontiguousarray(iq, dtype=np.int8)
        if iq.ndim == 1:
            iq = iq[None, :]
        ns, n = iq.shape
        ch = np.ascontiguousarray(np.broadcast_to(np.asarray(channels, dtype=np.int32), (ns,)))
        return self._grow_once(partial(self._L.btle_b200_discover, self._h, iq.ctypes.data, ns, n, n, ch.ctypes.data), CAND_DTYPE,
                               ns * (n // 16384 + 1) * 8 + 256 if cap is None else cap, grow=cap is None)

    # ---- unbounded capture, pushed in pieces (btle_b200_stream_*) -----------------------------
    def stream(self, segment_chunks: int = 0, **cfg) -> "RxStream":
        """Streaming session over one capture of any length: `with rx.stream(channel=37) as s: recs = s.push(iq_piece) ...;
        recs = s.finish()`.  Segments are double-buffered in page-locked memory; records come back in reference order,
        `chunk` counted from the start of the stream, as segments complete."""
        return RxStream(self, make_cfgs(1, **cfg), segment_chunks)

    def streams(self, cfgs: np.ndarray, segment_chunks: int = 0) -> "RxStreams":
        """Streaming session over N time-aligned captures (one per radio / channel), cfgs: CFG_DTYPE [N] (make_cfgs):
        `with rx.streams(make_cfgs(3, channel=[37, 38, 39])) as s: recs = s.push(1, iq_piece) ...; recs = s.finish()`.
        Equals rx_batch() on the captures cut to the shortest one.  Each segment set (segment_chunks chunks of every
        capture; 0 = the library default) is decoded in one batched launch once every capture has filled its part;
        records come back per set in (stream, chunk, n0) order, `chunk` counted from the start of the capture."""
        return RxStreams(self, cfgs, segment_chunks)

    # ---- device-resident ------------------------------------------------------------------
    def rx_device(self, d_iq, cfgs: np.ndarray, d_out, d_count, stream_ptr: int = 0):
        """d_iq: torch int8 CUDA tensor [n_streams, n_int8]; d_out: torch uint8 CUDA tensor
        [cap*64]; d_count: torch int32 CUDA tensor [1].  Enqueues on `stream_ptr` (no sync).  Records land in
        one block per unit of work (see include/btle_b200.h); sort_records() gives reference order."""
        ns, n = d_iq.shape
        cfgs = np.ascontiguousarray(cfgs, dtype=CFG_DTYPE)
        assert d_iq.stride(1) == 1 and cfgs.shape == (ns,)
        cap = d_out.numel() // 64
        rc = self._L.btle_b200_rx_device(self._h, d_iq.data_ptr(), ns, d_iq.stride(0), n, cfgs.ctypes.data,
                                         d_out.data_ptr(), cap, d_count.data_ptr(), ctypes.c_void_p(stream_ptr))
        self._check(rc)

    def discover_device(self, d_iq, channels, d_out, d_count, stream_ptr: int = 0):
        """d_iq: torch int8 CUDA tensor [n_streams, n_int8] (16-byte aligned rows); channels: the data channel of each row;
        d_out: torch CUDA tensor of cap * 32 bytes; d_count: torch int32 CUDA tensor [1].  Enqueues on `stream_ptr` (no
        sync).  Candidates land unordered in d_out[:min(count, cap)] (view the bytes as CAND_DTYPE)."""
        ns, n = d_iq.shape
        assert d_iq.stride(1) == 1
        ch = np.ascontiguousarray(np.broadcast_to(np.asarray(channels, dtype=np.int32), (ns,)))
        cap = d_out.numel() * d_out.element_size() // 32
        rc = self._L.btle_b200_discover_device(self._h, d_iq.data_ptr(), ns, d_iq.stride(0), n, ch.ctypes.data, d_out.data_ptr(), cap,
                                               d_count.data_ptr(), ctypes.c_void_p(stream_ptr))
        self._check(rc)

    def units(self, n_streams: int, n_int8: int) -> int:
        """Number of unit-directory entries a launch over this shape writes (btle_b200_rx_units)."""
        return int(self._L.btle_b200_rx_units(self._h, n_streams, n_int8))

    def rx_device_dir(self, d_iq, cfgs: np.ndarray, d_out, d_count, d_dir, stream_ptr: int = 0, offset_hz=None):
        """Like rx_device, with the unit directory in the caller's buffer: d_dir is a torch CUDA tensor of at least
        units(...) * 8 bytes.  d_out / d_dir may be views of PEER memory (another GPU's buffer mapped here): the kernel
        then stores records and directory straight over NVLink.  Walking the directory (gather_ordered) yields the
        records in the reference's order.  d_count may be None (the packet count is the sum of the directory's counts):
        no memset is then enqueued in front of the kernel.  offset_hz as rx_batch's (btle_b200_rx_device_dir_offset)."""
        ns, n = d_iq.shape
        cfgs = np.ascontiguousarray(cfgs, dtype=CFG_DTYPE)
        assert d_iq.stride(1) == 1 and cfgs.shape == (ns,)
        cap = d_out.numel() * d_out.element_size() // 64
        dir_cap = d_dir.numel() * d_dir.element_size() // 8
        off = _offsets(offset_hz, ns)
        self._check(self._L.btle_b200_rx_device_dir_offset(
            self._h, d_iq.data_ptr(), ns, d_iq.stride(0), n, cfgs.ctypes.data, _ptr(off), d_out.data_ptr(), cap,
            d_count.data_ptr() if d_count is not None else None, d_dir.data_ptr(), dir_cap, ctypes.c_void_p(stream_ptr)))

    def rec_offsets_device(self, d_iq, d_recs, n: int, d_hz, stream_ptr: int = 0):
        """rec_offsets on the device: d_iq as rx_device_dir's, d_recs n records (uint8 CUDA tensor of n * 64 bytes),
        d_hz float32 CUDA tensor [n]; enqueued on `stream_ptr` (no sync)."""
        ns, nb = d_iq.shape
        assert d_iq.stride(1) == 1 and d_hz.numel() >= n
        self._check(self._L.btle_b200_rec_offset_device(self._h, d_iq.data_ptr(), d_iq.stride(0), nb, d_recs.data_ptr(), n, d_hz.data_ptr(),
                                                        ctypes.c_void_p(stream_ptr)))

    def gather_ordered(self, recs: np.ndarray, unit_dir: np.ndarray) -> np.ndarray:
        """Host copies of a launch's record buffer and unit directory -> records in reference order."""
        recs = np.ascontiguousarray(recs, dtype=REC_DTYPE)
        unit_dir = np.ascontiguousarray(unit_dir, dtype=DIR_DTYPE)
        total = int(unit_dir["count"].sum())
        out = np.empty(total, dtype=REC_DTYPE)
        n_out = ctypes.c_size_t(0)
        rc = self._L.btle_b200_gather_ordered(recs.ctypes.data, recs.size, unit_dir.ctypes.data, unit_dir.size, out.ctypes.data,
                                              total, ctypes.byref(n_out))
        if rc != 0:
            raise BtleError(rc, "record buffer holds fewer records than the directory describes (capacity overflow)")
        return out

    def sort_records(self, recs: np.ndarray) -> np.ndarray:
        recs = np.ascontiguousarray(recs, dtype=REC_DTYPE)
        self._L.btle_b200_sort_records(recs.ctypes.data, recs.size)
        return recs

    # ---- leaf functions with the reference's signatures ----------------------------------
    def search_unique_bits(self, rxp: np.ndarray, search_len: int, unique_bits, unique_bits_mask, num_bits=32) -> int:
        rxp = np.ascontiguousarray(rxp, dtype=np.int8)
        assert rxp.size >= 8 * search_len + 2
        ub = np.ascontiguousarray(unique_bits, dtype=np.uint8)
        um = np.ascontiguousarray(unique_bits_mask, dtype=np.uint8)
        r = self._L.btle_b200_search_unique_bits(self._h, rxp.ctypes.data, search_len, ub.ctypes.data, um.ctypes.data, num_bits)
        if r <= -1000:                     # BTLE_SEARCH_ERR(code): errors live below every possible hit index
            self._check(r + 1000)
        return r

    def demod_byte(self, rxp: np.ndarray, num_byte: int) -> np.ndarray:
        rxp = np.ascontiguousarray(rxp, dtype=np.int8)
        out = np.zeros(num_byte, dtype=np.uint8)
        self._check(self._L.btle_b200_demod_byte(self._h, rxp.ctypes.data, num_byte, out.ctypes.data))
        return out

    def scramble_byte(self, byte_in, channel: int, table_offset: int = 0) -> np.ndarray:
        b = np.ascontiguousarray(byte_in, dtype=np.uint8)
        out = np.zeros_like(b)
        self._check(self._L.btle_b200_scramble_byte(self._h, b.ctypes.data, b.size, channel, table_offset, out.ctypes.data))
        return out

    def crc24_byte(self, byte_in, init_hex: int) -> int:
        b = np.ascontiguousarray(byte_in, dtype=np.uint8)
        out = ctypes.c_uint32(0)
        self._check(self._L.btle_b200_crc24_byte(self._h, b.ctypes.data, b.size, init_hex, ctypes.byref(out)))
        return out.value

    def crc_init_reorder(self, crc_init: int) -> int:
        return self._L.btle_b200_crc_init_reorder(crc_init)

    def dbits(self, iq: np.ndarray) -> np.ndarray:
        iq = np.ascontiguousarray(iq, dtype=np.int8)
        n = iq.size // 2 - 1
        out = np.zeros(max(n, 0), dtype=np.uint8)
        if n > 0:
            self._check(self._L.btle_b200_dbits(self._h, iq.ctypes.data, n, out.ctypes.data))
        return out


class RxStream:
    """Python face of btle_b200_stream_open / push / finish / close."""

    def __init__(self, rx: BtleRx, cfgs: np.ndarray, segment_chunks: int):
        self._rx, self._L = rx, rx._L
        self._cfg = np.ascontiguousarray(cfgs, dtype=CFG_DTYPE)
        h = ctypes.c_void_p()
        rx._check(self._L.btle_b200_stream_open(rx._h, self._cfg.ctypes.data, int(segment_chunks), ctypes.byref(h)))
        self._h = h
        self._buf = np.empty(65536, dtype=REC_DTYPE)

    def push(self, iq) -> np.ndarray:
        iq = np.ascontiguousarray(iq, dtype=np.int8).reshape(-1)
        out, done, step = [], 0, 64 << 20
        while done < iq.size:                   # a push never returns more records than the buffer holds: feed it in bounded pieces
            piece = iq[done:done + step]
            n = ctypes.c_size_t(0)
            self._rx._check(self._L.btle_b200_stream_push(self._h, piece.ctypes.data, piece.size, self._buf.ctypes.data, self._buf.size, ctypes.byref(n)))
            out.append(self._buf[:n.value].copy())
            done += piece.size
        return np.concatenate(out) if out else self._buf[:0].copy()

    def finish(self) -> np.ndarray:
        return self._rx._drain(self._L.btle_b200_stream_finish, self._h, self._buf)

    def set_offset(self, offset_hz: float) -> None:
        """Carrier-offset correction of the capture from the next submitted segment on (btle_b200_stream_set_offset)."""
        self._rx._check(self._L.btle_b200_stream_set_offset(self._h, float(offset_hz)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.btle_b200_stream_close(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    __del__ = close


class RxStreams:
    """Python face of btle_b200_streams_open / acquire / commit / set_cfg / finish / close.

    push(stream, iq) never blocks: bytes of a capture whose part of the current segment set is complete (the session waits
    for the other captures) are kept here and fed in as soon as that set has been handed to the GPU."""

    def __init__(self, rx: BtleRx, cfgs: np.ndarray, segment_chunks: int):
        self._rx, self._L = rx, rx._L
        self._cfgs = np.array(cfgs, dtype=CFG_DTYPE).reshape(-1)
        self.n_streams = int(self._cfgs.size)
        h = ctypes.c_void_p()
        rx._check(self._L.btle_b200_streams_open(rx._h, self._cfgs.ctypes.data if self.n_streams else None, self.n_streams,
                                                 int(segment_chunks), ctypes.byref(h)))
        self._h = h
        self._buf = np.empty(65536, dtype=REC_DTYPE)
        self._pending = [[] for _ in range(self.n_streams)]     # per capture: arrays not yet taken by the session

    def _acquire(self, stream):
        buf, space = ctypes.c_void_p(), ctypes.c_size_t(0)
        self._rx._check(self._L.btle_b200_streams_acquire(self._h, stream, ctypes.byref(buf), ctypes.byref(space)))
        return buf.value, space.value

    def _commit(self, stream, n_int8, out):
        n = ctypes.c_size_t(0)
        self._rx._check(self._L.btle_b200_streams_commit(self._h, stream, n_int8, self._buf.ctypes.data, self._buf.size, ctypes.byref(n)))
        out.append(self._buf[:n.value].copy())
        while n.value == self._buf.size:        # more records waiting than the buffer holds
            self._rx._check(self._L.btle_b200_streams_commit(self._h, stream, 0, self._buf.ctypes.data, self._buf.size, ctypes.byref(n)))
            out.append(self._buf[:n.value].copy())

    def push(self, stream: int, iq) -> np.ndarray:
        """Append bytes to capture `stream`; returns the records of the segment sets completed so far."""
        stream = int(stream)
        self._acquire(stream)                   # BtleError (BTLE_EINVAL) for an index out of range
        iq = np.ascontiguousarray(iq, dtype=np.int8).reshape(-1)
        if iq.size:
            self._pending[stream].append(iq)
        out, progress = [], True
        while progress:                         # completing a set frees room for every capture's waiting bytes
            progress = False
            for i, q in enumerate(self._pending):
                while q:
                    buf, space = self._acquire(i)
                    if space == 0:
                        break
                    k = min(space, q[0].size)
                    ctypes.memmove(buf, q[0].ctypes.data, k)
                    q[0] = q[0][k:]
                    if q[0].size == 0:
                        q.pop(0)
                    self._commit(i, k, out)
                    progress = True
        q = self._pending[stream]
        if q and np.may_share_memory(q[-1], iq):     # keep what waits independent of the caller's array
            q[-1] = q[-1].copy()
        return np.concatenate(out) if out else self._buf[:0].copy()

    def set_cfg(self, stream: int, **cfg) -> None:
        """Change fields of capture `stream`'s cfg (make_cfgs names), from the next segment set that is submitted on."""
        c = _with_fields(self._cfgs[int(stream):int(stream) + 1].copy() if 0 <= int(stream) < self.n_streams else make_cfgs(1), cfg)
        self._rx._check(self._L.btle_b200_streams_set_cfg(self._h, int(stream), c.ctypes.data))
        self._cfgs[int(stream)] = c[0]

    def set_offset(self, stream: int, offset_hz: float) -> None:
        """Carrier-offset correction of capture `stream` (Hz, received minus nominal carrier), from the next segment set
        that is submitted on; from the first call on, every set takes the rotated kernel (btle_b200_streams_set_offset)."""
        self._rx._check(self._L.btle_b200_streams_set_offset(self._h, int(stream), float(offset_hz)))

    # ---- per-capture cfg lists and discovery (btle_b200_streams_add_cfg / remove_cfg / set_discover) -------------------
    @property
    def resident(self) -> int:
        """First chunk of the oldest segment set still on the device: the smallest from_chunk add_cfg() accepts."""
        v = ctypes.c_int64(0)
        self._rx._check(self._L.btle_b200_streams_resident(self._h, ctypes.byref(v)))
        return v.value

    def add_cfg(self, capture: int, from_chunk: int | None = None, **cfg) -> tuple:
        """One more cfg on capture `capture`: capture's own cfg with the given fields (make_cfgs names) changed, decoding
        chunks >= from_chunk (None: `resident`, so the sets still on the device are decoded with it too).  Returns
        (index, from_chunk); records of this cfg carry `stream` = index.  Records of resident sets come back from the
        next push() or finish()."""
        capture = int(capture)
        c = _with_fields(self._cfgs[capture:capture + 1].copy() if 0 <= capture < self.n_streams else make_cfgs(1), cfg)
        frm = self.resident if from_chunk is None else int(from_chunk)
        idx = ctypes.c_size_t(0)
        self._rx._check(self._L.btle_b200_streams_add_cfg(self._h, capture, c.ctypes.data, frm, ctypes.byref(idx)))
        return idx.value, frm

    def remove_cfg(self, index: int) -> int:
        """Cfg `index` decodes no chunk from the next submitted segment set on; returns that set's first chunk."""
        v = ctypes.c_int64(0)
        self._rx._check(self._L.btle_b200_streams_remove_cfg(self._h, int(index), ctypes.byref(v)))
        return v.value

    def set_discover(self, channels) -> None:
        """channels[i]: data channel 0..36 scanned for connection candidates on capture i, or -1; from the next set on."""
        ch = np.ascontiguousarray(np.broadcast_to(np.asarray(channels, dtype=np.int32), (self.n_streams,)))
        self._rx._check(self._L.btle_b200_streams_set_discover(self._h, ch.ctypes.data))

    def candidates(self) -> np.ndarray:
        """Discovery candidates (CAND_DTYPE) of the sets handed out since the last call, per set by (stream, sample);
        `sample` counted from the capture's start, `stream` = capture index."""
        buf = np.empty(16384, dtype=CAND_DTYPE)
        return self._rx._drain(self._L.btle_b200_streams_take_cands, self._h, buf)

    def finish(self) -> np.ndarray:
        """End of the captures: decodes up to the shortest one and returns every record still waiting."""
        out = self._rx._drain(self._L.btle_b200_streams_finish, self._h, self._buf)
        self._pending = [[] for _ in range(self.n_streams)]   # bytes behind the shortest capture are not decoded
        return out

    def close(self):
        if getattr(self, "_h", None):
            self._L.btle_b200_streams_close(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    __del__ = close
