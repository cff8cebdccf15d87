"""Offline connection following across concurrently captured BLE channels (SURVEY.md §8f-2).

The reference follows ONE connection in real time by retuning its single radio
(`receiver_controller`, host/btle-tools/src/btle_rx.c:2403-2536): after a CRC-ok CONNECT_REQ with
a full channel map it takes the access address, CRCInit, hop increment and interval from the
payload (`parse_adv_pdu_payload_byte`, :1617-1698), jumps to data channel `hop % 37`, waits for
the first CRC-ok data packet, and from then on hops `(chan + hop) % 37` once per connection
interval (guard 7 ms before, "skip" after interval - 4 ms without a packet).

With all 40 channels captured at once nothing has to be retuned, and EVERY connection can be followed (the
reference's single radio follows the first one; that exact behaviour is `btle_rx_b200 -o --iq-dir`, built on the C state
machine `btle_b200_receiver_controller`).  follow_connections(): pass 1 decodes the advertising channels, pass 2 re-runs the
receive kernel over the 37 data-channel captures once per connection with that connection's access address / CRCInit, and
the hop sequence is used to attribute each data packet to a connection event.  follow_connections_windowed(): the same
result from three batched launches in total — only the windows the virtual radio of each connection would dwell in are
decoded (about two single-channel passes per connection instead of 37).  Same rules as the reference: only full channel maps
(`chm_is_full_map`, :2395-2400) are tracked, others are reported as dropped.
discover_connections(): connections whose CONNECT_REQ was not captured, found from the empty PDUs on the data channels
(the GPU candidate scan BtleRx.discover); follow_connections(discover=True) follows them as well."""
from __future__ import annotations

import numpy as np

from .rx import make_cfgs

SAMPLE_RATE = 4.0e6
GUARD_US = 7000          # btle_rx.c:2404
SKIP_GUARD_US = 4000     # btle_rx.c:2405


def record_time(rec) -> float:
    """Seconds from the start of the capture to the first access-address sample."""
    return (int(rec["chunk"]) * 8192 + int(rec["n0"])) / SAMPLE_RATE


def _ll_data_fields(p: bytes) -> dict:
    """The 34-byte payload of a CONNECT_IND / AUX_CONNECT_REQ (InitA, AdvA, LLData) as the reference reads it."""
    return {
        "init_a": p[0:6][::-1].hex(), "adv_a": p[6:12][::-1].hex(),
        "access_addr": int.from_bytes(p[12:16], "little"),
        "crc_init": (p[16] << 16) | (p[17] << 8) | p[18],          # as the reference reads it, :1637-1639
        "win_size": p[19], "win_offset": int.from_bytes(p[20:22], "little"),
        "interval": int.from_bytes(p[22:24], "little"), "latency": int.from_bytes(p[24:26], "little"),
        "timeout": int.from_bytes(p[26:28], "little"), "chm": p[28:33][::-1].hex(),
        "hop": p[33] & 0x1F, "sca": (p[33] >> 5) & 7,
    }


def parse_connect_req(rec):
    """Fields the reference keeps in `receiver_status` (btle_rx.c:1683-1698), or None."""
    b = rec["bytes"]
    if rec["crc_bad"] or (b[0] & 0x0F) != 5 or (b[1] & 0x3F) != 34:
        return None
    return {"t": record_time(rec), "adv_channel": int(rec["channel"]), **_ll_data_fields(bytes(b[2:36]))}


AUX_CONNECT_REQ = 5          # PDU type of AUX_CONNECT_REQ on a secondary advertising channel (Core Spec Vol 6 Part B §2.3)


def parse_aux_connect_req(rec):
    """An LE Coded PHY record (CODED_REC_DTYPE) of an AUX_CONNECT_REQ -> parse_connect_req()'s fields plus "aux": True, or
    None.  AUX_CONNECT_REQ carries the same InitA, AdvA and LLData as CONNECT_IND (Core Spec Vol 6 Part B §2.3.3.2); its
    length field is 8 bits.  `t` is the record's sample / 4 Msps and `adv_channel` the secondary channel it came on."""
    b = rec["bytes"]
    if rec["crc_bad"] or (b[0] & 0x0F) != AUX_CONNECT_REQ or b[1] != 34:
        return None
    return {"t": int(rec["sample"]) / SAMPLE_RATE, "adv_channel": int(rec["channel"]), **_ll_data_fields(bytes(b[2:36])), "aux": True}


def new_connections(conns, found):
    """found without the connections whose (access address, CRC init) is already in conns or earlier in found."""
    seen = {(c["access_addr"], c["crc_init"]) for c in conns}
    out = []
    for c in found:
        key = (c["access_addr"], c["crc_init"])
        if key not in seen:
            seen.add(key)
            out.append(c)
    return out


def connection_cfgs(batch, **flags):
    """The cfgs and capture list of one several-cfgs-per-capture call over the data captures 0..36 for up to
    MAX_CFGS_PER_CAPTURE connections: cfg j = channel * k + i is connection i on data channel j // k (the cfgs of one
    capture are adjacent), so a record's connection is stream % k.  flags: make_cfgs() keywords for every cfg."""
    k = len(batch)
    cfgs = make_cfgs(37 * k, channel=np.repeat(np.arange(37), k), access_addr=[c["access_addr"] for c in batch] * 37,
                     crc_init=[c["crc_init"] for c in batch] * 37, **flags)
    return cfgs, np.repeat(np.arange(37, dtype=np.int32), k)


def _walk_events(c, per_ch, n_samples, max_events=10000, first_channel=None):
    """The reference's state machine (states 1-3 of receiver_controller, btle_rx.c:2455-2530) over per-channel lists of
    the connection's data-channel records.  Returns (events, queries): queries = the (channel, t_lo, t_hi) ranges the walk
    looked at, so that a caller that decoded only windows can verify it had decoded all of them.  The walk waits from
    c["t"] on its first channel: hop % 37 as after a CONNECT_REQ, or `first_channel` (a discovered connection)."""
    interval_s = c["interval"] * 1250e-6                                                  # :2430
    chan = 0 if first_channel is None else (first_channel - c["hop"]) % 37
    events, queries, t_mark, anchored = [], [], None, True
    for k in range(max_events):
        chan = (chan + c["hop"]) % 37                                                     # :2434 / :2476
        pk = per_ch[chan]
        if t_mark is None:                       # state 1: wait for the first CRC-ok data packet
            first = next((r for r in pk if not r["crc_bad"]), None)
            if first is None:
                queries.append((chan, c["t"], float("inf")))
                break
            t_ev, t_hop, now_anchored = record_time(first), c["t"], True
            got = [r for r in pk if t_ev <= record_time(r) < t_ev + interval_s - GUARD_US * 1e-6]
            queries.append((chan, c["t"], t_ev + interval_s - GUARD_US * 1e-6))
        else:
            # state 2 -> 3: the hop happens `interval - 7 ms` after the mark of an event that saw a packet (:2472);
            # after a "skip" the reference is already on the next channel at the skip instant (:2504-2522), the mark
            # IS that instant.  In state 3 the channel is left `interval - 4 ms` after the mark without a packet.
            lo = t_mark + (interval_s - GUARD_US * 1e-6 if anchored else 0.0)
            hi = (lo if anchored else t_mark) + interval_s - SKIP_GUARD_US * 1e-6
            got = [r for r in pk if lo <= record_time(r) < hi]
            queries.append((chan, lo, hi))
            ok = next((r for r in got if not r["crc_bad"]), None)
            t_ev = record_time(ok) if ok is not None else hi                              # "Hop: skip": mark = skip instant
            t_hop, now_anchored = lo, ok is not None
            if t_ev * SAMPLE_RATE > n_samples:
                break
        # t_hop: when the reference would have retuned to this channel; anchored: a CRC-ok packet was seen on it
        events.append({"k": k, "channel": chan, "t": t_ev, "t_hop": t_hop, "anchored": now_anchored, "packets": got})
        t_mark, anchored = t_ev, now_anchored
    return events, queries


def _pre_s(interval_s: float) -> float:
    """How far before the ideal event time t_first + k*interval a window starts.  After an event that saw a packet the
    reference arrives 7 ms early; after a missed event ("skip") it is already there 11 ms early, and every further consecutive
    miss adds 4 ms (btle_rx.c:2404-2405, :2504-2522): room for three misses in a row, more fall back to full passes."""
    return max(0.5 * interval_s, 0.011 + 2 * 0.004 + 0.001)


def _rx_windows(rx, captures, windows, w_chunks):
    """windows: list of (channel, first chunk, cfg dict).  Decodes w_chunks chunks of every window in ONE batched launch
    (windows are gathered into a staging batch with their look-ahead; bytes behind a capture are zero).  Returns the records
    with `stream` = window index and `chunk` = absolute chunk index in the capture."""
    n = captures.shape[1]
    length = w_chunks * 16384 + 4096
    stage = np.zeros((len(windows), length), dtype=np.int8)
    cfgs = make_cfgs(len(windows))
    for i, (ch, k0, cfg) in enumerate(windows):
        a = k0 * 16384
        seg = captures[ch, a:min(n, a + length)]
        stage[i, :seg.size] = seg
        cfgs[i]["channel"], cfgs[i]["access_addr"], cfgs[i]["crc_init"] = ch, cfg["access_addr"], cfg["crc_init"]
    rec = rx.rx_batch(stage, cfgs).copy()
    nchunks = n // 16384
    k0s = np.array([w[1] for w in windows], dtype=np.int64)
    rec["chunk"] += k0s[rec["stream"]].astype(np.int32)
    return rec[rec["chunk"] < nchunks]                       # a window may reach behind the last complete chunk of the capture


def follow_connections_windowed(rx, captures: np.ndarray, first_search_chunks: int = 48, max_events: int = 10000):
    """follow_connections() for MANY connections at the cost of about two single-channel passes per connection instead of
    37: three batched launches in total, whatever the number of CONNECT_REQs.
      1. the three advertising captures -> CONNECT_REQs;
      2. per tracked connection one window of `first_search_chunks` chunks on its first data channel behind the CONNECT_REQ
         -> the first CRC-ok data packet (the anchor of state 1);
      3. per connection event k one window on channel (k+1)*hop % 37 covering the whole dwell the reference's radio would
         spend there, predicted from the anchor (t_first + k*interval): from 20 ms (or half an interval) before the ideal
         event time to a full interval behind it (missed events move the reference's hop times earlier by up to 4 ms each).
    The state-machine walk then runs on what the windows returned and reports the time ranges it looked at; a connection
    whose walk looked outside its decoded windows (long runs of skips) is redone with full data-channel passes.  Same
    return value as follow_connections(), plus conn["chunks_decoded"]."""
    captures = np.ascontiguousarray(captures, dtype=np.int8)
    assert captures.shape[0] == 40
    n = captures.shape[1]
    nchunks = n // 16384
    adv = rx.rx_batch(captures[37:40], make_cfgs(3, channel=[37, 38, 39])).copy()
    adv["stream"] += 37
    conns = []
    for r in adv:
        c = parse_connect_req(r)
        if c is None:
            continue
        c["tracked"] = c["chm"] == "1fffffffff" and c["interval"] > 0
        conns.append(c)
    live = [c for c in conns if c["tracked"]]
    if not live:
        return adv, conns
    chunk_of = lambda t: int(t * SAMPLE_RATE) // 8192
    # 2. anchors
    F = max(1, min(first_search_chunks, nchunks))
    w1 = [(c["hop"] % 37, min(chunk_of(c["t"]), max(0, nchunks - 1)), c) for c in live]
    rec1 = _rx_windows(rx, captures, w1, F)
    for i, c in enumerate(live):
        mine = rec1[rec1["stream"] == i]
        ok = [r for r in mine if not r["crc_bad"] and record_time(r) > c["t"]]
        c["_anchor"] = record_time(ok[0]) if ok else None
        c["_recs"] = [mine]
        c["_cover"] = {c["hop"] % 37: [(w1[i][1], w1[i][1] + F)]}
    # 3. every event of every connection
    w2, owner, W = [], [], 1
    for c in live:
        if c["_anchor"] is None:
            continue
        interval_s = c["interval"] * 1250e-6
        W = max(W, int(np.ceil((_pre_s(interval_s) + interval_s) * SAMPLE_RATE / 8192)) + 2)
    for ci, c in enumerate(live):
        if c["_anchor"] is None:
            continue
        interval_s = c["interval"] * 1250e-6
        chan, e = c["hop"] % 37, 0
        while e < max_events:
            e += 1
            chan = (chan + c["hop"]) % 37
            t_e = c["_anchor"] + e * interval_s
            if t_e - interval_s > n / 2 / SAMPLE_RATE:
                break
            k0 = max(0, chunk_of(t_e - _pre_s(interval_s)) - 1)
            if k0 >= nchunks:
                break
            w2.append((chan, k0, c))
            owner.append(ci)
            c["_cover"].setdefault(chan, []).append((k0, k0 + W))
    if w2:
        rec2 = _rx_windows(rx, captures, w2, W)
        owner = np.array(owner)
        for ci, c in enumerate(live):
            sel = np.nonzero(owner == ci)[0]
            if len(sel):
                c["_recs"].append(rec2[np.isin(rec2["stream"], sel)])
    for c in live:
        allr = np.concatenate(c["_recs"])
        # windows overlap: a packet decoded twice is one packet
        key = allr["channel"].astype(np.int64) * (1 << 40) + allr["chunk"].astype(np.int64) * (1 << 16) + (allr["n0"].astype(np.int64) + 1024)
        _, first_idx = np.unique(key, return_index=True)
        allr = allr[np.sort(first_idx)]
        allr = allr[np.argsort(allr["chunk"].astype(np.int64) * 8192 + allr["n0"], kind="stable")]
        per_ch = {ch: [] for ch in range(37)}
        for r in allr:
            if record_time(r) > c["t"]:
                per_ch[int(r["channel"])].append(r)
        events, queries = _walk_events(c, per_ch, n // 2, max_events)
        c["chunks_decoded"] = int(sum(b - a for v in c["_cover"].values() for a, b in v))
        covered = True
        t_end = n / 2 / SAMPLE_RATE
        for ch, lo, hi in queries:
            ka, kb = chunk_of(max(lo, 0.0)), min(nchunks, chunk_of(min(hi, t_end)) + 1)
            need = set(range(ka, kb))
            for a, b in c["_cover"].get(ch, []):
                need -= set(range(a, b))
            if need:
                covered = False
                break
        if not covered:                          # the walk left the predicted windows: decode this connection's data channels in full
            cfgs = make_cfgs(37, channel=list(range(37)), access_addr=c["access_addr"], crc_init=c["crc_init"])
            data = rx.rx_batch(captures[0:37], cfgs)
            per_ch = {ch: [] for ch in range(37)}
            for r in data:
                if record_time(r) > c["t"]:
                    per_ch[int(r["channel"])].append(r)
            events, _ = _walk_events(c, per_ch, n // 2, max_events)
            c["chunks_decoded"] += 37 * nchunks
        c["events"] = events
        for k_ in ("_anchor", "_recs", "_cover"):
            c.pop(k_, None)
    return adv, conns


def follow_connections(rx, captures: np.ndarray, max_events: int = 10000, discover: bool = False):
    """captures: int8 [40, n_int8], row c = BLE channel c, all rows time-aligned.
    `rx` needs `rx_batch(iq, cfgs)` (a BtleRx).  Returns (adv_records, connections) where each
    connection is the parse_connect_req dict plus `tracked`, and, if tracked, `events`: a list of
    {"k", "channel", "t", "packets"} with `packets` the data-channel records of that event.
    discover=True (`rx` then also needs `discover(iq, channels)`): the connections discover_connections() finds on the
    data channels are appended, and every tracked one whose access address is not that of a tracked CONNECT_REQ is
    followed the same way, its walk starting on `first_channel` 1.25 ms before `t_first` (so that a master packet in
    front of the first empty PDU anchors it)."""
    captures = np.ascontiguousarray(captures, dtype=np.int8)
    assert captures.shape[0] == 40
    adv = rx.rx_batch(captures[37:40], make_cfgs(3, channel=[37, 38, 39]))
    adv = adv.copy()
    adv["stream"] += 37
    conns = []
    for r in adv:
        c = parse_connect_req(r)
        if c is None:
            continue
        # :2417 full channel map only.  (interval == 0 would make the reference hop on every chunk; such a CONNECT_REQ is
        # reported as not tracked here — a deliberate difference.)
        c["tracked"] = c["chm"] == "1fffffffff" and c["interval"] > 0
        conns.append(c)
    walks = [(c, c, None) for c in conns if c["tracked"]]
    if discover:
        known = {c["access_addr"] for c in conns if c["tracked"]}
        found = discover_connections(rx, captures)
        conns += found
        walks += [(c, dict(c, t=c["t_first"] - DISCOVER_LEAD_S), c["first_channel"]) for c in found
                  if c["tracked"] and c["access_addr"] not in known]
    for c, walk, first_channel in walks:
        cfgs = make_cfgs(37, channel=list(range(37)), access_addr=c["access_addr"], crc_init=c["crc_init"])
        data = rx.rx_batch(captures[0:37], cfgs)
        per_ch = {ch: [] for ch in range(37)}
        for r in data:
            if record_time(r) > walk["t"]:
                per_ch[int(r["channel"])].append(r)
        c["events"] = _walk_events(walk, per_ch, captures.shape[1] // 2, max_events, first_channel)[0]
    return adv, conns


def decode_connections(rx, captures: np.ndarray, discover: bool = True, offset_hz=None, symbol_spaced: bool = False,
                       centre_hits: bool = False, correct: bool = False, lowpass: bool = False, offset_search: bool = False,
                       coded: bool = False, coded_discover: bool = False):
    """Every known connection's data-channel traffic, decoded without following it.  captures: int8 [40, n_int8] as in
    follow_connections(); `rx` needs rx_batch, rx_multi, with discover=True discover, and with coded=True rx_coded and
    rx_coded_multi (a BtleRx).
    The connections are the CONNECT_REQ ones (tracked or not) plus, with discover=True, the discover_connections() ones
    whose access address no CONNECT_REQ announced (tracked or not: a partial channel map or CSA#2 does not matter here).
    With all 37 data channels captured, a connection's packets are found by its access address and CRC init alone, so
    each connection gets `traffic`: every record on channels 0..36 decoded with them, in time order (chunk * 8192 + n0,
    then channel).  Launches: one rx_batch over the advertising captures, one discover, and one rx_multi per
    MAX_CFGS_PER_CAPTURE connections over captures[0:37] (each capture is read once per call, whatever the number of
    connections in it).  offset_hz (a scalar or one per capture, None: no correction) is passed to those rx_batch and
    rx_multi calls (carrier-offset correction); discovery reads the captures uncorrected.  symbol_spaced: every receive
    cfg of those calls carries BTLE_CFG_SYMBOL_SPACED (the symbol-spaced discriminator); centre_hits: every receive cfg of
    those calls carries BTLE_CFG_CENTRE_HITS (each hit centred on its run of matching sample phases); correct: every
    receive cfg of those calls carries BTLE_CFG_CORRECT (one-bit and adjacent-pair errors corrected from the CRC
    syndrome); lowpass: every receive cfg of those calls carries BTLE_CFG_LOWPASS (the symbol-spaced bits of [1, 2, 1]
    filtered samples; only with symbol_spaced); offset_search: every receive cfg of those calls carries BTLE_CFG_OFFSET_SEARCH
    (seven carrier-offset hypotheses per capture, merged per packet); discovery keeps its own rule.
    coded=True adds the LE Coded PHY, in 1 + ceil(connections / MAX_CFGS_PER_CAPTURE) more launches:
      - one rx_coded over captures[0:37] with the advertising access address and CRC init on each capture's channel: its
        CRC-ok AUX_CONNECT_REQs (parse_aux_connect_req) become connections with "aux": True and `tracked` False (they use
        CSA#2), after those whose (access address, CRC init) is already known;
      - one rx_coded_multi per MAX_CFGS_PER_CAPTURE connections (every connection, AUX_CONNECT_REQ ones included) over
        captures[0:37], cfgs laid out as for rx_multi: each connection gets `coded_traffic`, its coded records (stream =
        channel) in (sample, channel) order.  So a 1M connection that moved to the coded PHY is covered too.
    offset_hz is passed to the coded calls as well; the 1M opt-in flags are not (the coded receiver has none).  AUX_CONNECT_REQ
    connections get `traffic` like every other one.  With coded=False the result is what it was without the argument.
    coded_discover=True (with coded=True; `rx` then also needs discover_coded) adds one discover_coded call over
    captures[0:37] after the rx_coded one: the discover_coded_connections() connections whose (access address, CRC init)
    is not already known are added after the AUX_CONNECT_REQ ones, and get `traffic` and `coded_traffic` like every other
    connection.  With coded_discover=False the result and the calls are what they were without the argument.
    Returns (adv_records, connections)."""
    from ._native import MAX_CFGS_PER_CAPTURE
    captures = np.ascontiguousarray(captures, dtype=np.int8)
    assert captures.shape[0] == 40
    # offsets are only passed when given: `rx` may be any object with BtleRx's rx_batch / rx_multi
    off = None if offset_hz is None else np.broadcast_to(np.asarray(offset_hz, dtype=np.float32), (40,))
    adv_kw = {} if off is None else {"offset_hz": off[37:40]}
    data_kw = {} if off is None else {"offset_hz": off[0:37]}
    flags = dict(symbol_spaced=symbol_spaced, centre_hits=centre_hits, correct=correct, lowpass=lowpass, offset_search=offset_search)
    adv = rx.rx_batch(captures[37:40], make_cfgs(3, channel=[37, 38, 39], **flags), **adv_kw).copy()
    adv["stream"] += 37
    conns = []
    for r in adv:
        c = parse_connect_req(r)
        if c is None:
            continue
        c["tracked"] = c["chm"] == "1fffffffff" and c["interval"] > 0
        conns.append(c)
    if discover:
        announced = {c["access_addr"] for c in conns}
        conns += [c for c in discover_connections(rx, captures) if c["access_addr"] not in announced]
    if coded:
        sec = rx.rx_coded(captures[0:37], make_cfgs(37, channel=list(range(37))), **data_kw)
        aux = [c for c in (parse_aux_connect_req(r) for r in sec) if c is not None]
        for c in aux:
            c["tracked"] = False
        conns += new_connections(conns, aux)
        if coded_discover:
            conns += new_connections(conns, discover_coded_connections(rx, captures, offset_hz=off))
    K = MAX_CFGS_PER_CAPTURE
    for b0 in range(0, len(conns), K):
        batch = conns[b0:b0 + K]
        k = len(batch)
        cfgs, capture = connection_cfgs(batch, **flags)
        rec = rx.rx_multi(captures[0:37], cfgs, capture, **data_kw)
        owner = rec["stream"] % k
        t = rec["chunk"].astype(np.int64) * 8192 + rec["n0"]
        for i, c in enumerate(batch):
            mine = rec[owner == i]
            tm = t[owner == i]
            tr = mine[np.lexsort((mine["channel"], tm))].copy()
            tr["stream"] = tr["channel"]                 # the capture row, as in follow_connections()
            c["traffic"] = tr
    if coded:
        for b0 in range(0, len(conns), K):
            batch = conns[b0:b0 + K]
            k = len(batch)
            cfgs, capture = connection_cfgs(batch)
            rec = rx.rx_coded_multi(captures[0:37], cfgs, capture, **data_kw)
            owner = rec["stream"] % k
            for i, c in enumerate(batch):
                mine = rec[owner == i]
                tr = mine[np.lexsort((mine["channel"], mine["sample"]))].copy()
                tr["stream"] = tr["channel"]
                c["coded_traffic"] = tr
    return adv, conns


# ---- connections whose CONNECT_REQ was not captured (DESIGN.md §6.2) ----------------------------------------------------
EVENT_SPAN_S = 3.75e-3   # candidates on one channel within half the shortest interval (7.5 ms) of the first are one event
DISCOVER_LEAD_S = 1.25e-3   # a discovered connection's walk starts this long before its first empty PDU


def _connection_from_events(aa, crc_init, events, n_candidates):
    """events: [(t, channel)] in time order -> the discovered-connection dict.  The interval is the GCD of the gaps
    between consecutive events in 1.25 ms units; with CSA#1 and a full channel map ch' = ch + hop (mod 37) per interval,
    so a gap of m intervals gives hop = dch * m^-1 (mod 37).  `tracked` only if the interval lies in 6..3200 and every
    pair gives the same non-zero hop; otherwise (a partial channel map, CSA#2) interval / hop are None."""
    units = [int(round((b[0] - a[0]) / 1.25e-3)) for a, b in zip(events, events[1:])]
    interval, hop = 0, None
    for u in units:
        interval = int(np.gcd(interval, u))
    ok = 6 <= interval <= 3200
    if ok:
        hops = set()
        for (_, ca), (_, cb), u in zip(events, events[1:], units):
            m = (u // interval) % 37
            if m == 0:                            # 37k intervals: back on the same channel, no information on the hop
                ok = ok and ca == cb
                continue
            hops.add((cb - ca) * pow(m, -1, 37) % 37)
        ok = ok and len(hops) == 1 and 0 not in hops
        hop = hops.pop() if ok else None
    return {"access_addr": aa, "crc_init": crc_init, "hop": hop, "interval": interval if ok else None, "chm": "1fffffffff",
            "t_first": events[0][0], "first_channel": events[0][1], "n_events": len(events), "n_candidates": n_candidates,
            "discovered": True, "adv_channel": None, "init_a": None, "adv_a": None, "tracked": ok}


def discover_connections(rx, captures: np.ndarray, min_events: int = 4):
    """Connections found from their empty PDUs alone, without a CONNECT_REQ.  captures: int8 [40, n_int8] as in
    follow_connections(); rows 0..36 are scanned in one rx.discover() call.  Candidates are grouped by (access address,
    CRC init); in a group, sorted by sample, candidates on the channel of the current event within 3.75 ms of its first
    candidate belong to it, any other starts the next event (time = first candidate's sample / 4 Msps).  Groups with fewer
    than `min_events` events are noise and are dropped.  Returns the _connection_from_events() dicts in order of t_first."""
    captures = np.ascontiguousarray(captures, dtype=np.int8)
    assert captures.shape[0] == 40
    return _group_candidates(rx.discover(captures[0:37], np.arange(37, dtype=np.int32)), min_events)


def _group_candidates(cand, min_events: int):
    """discover_connections()' grouping of candidates (any record with sample, access_addr, crc_init and channel) into
    _connection_from_events() dicts in order of t_first"""
    if len(cand) == 0:
        return []
    cand = cand[np.lexsort((cand["sample"], cand["crc_init"], cand["access_addr"]))]
    key = cand["access_addr"].astype(np.int64) << 24 | cand["crc_init"].astype(np.int64)
    cuts = np.flatnonzero(np.diff(key)) + 1
    conns = []
    for grp in np.split(cand, cuts):
        events = []
        for r in grp:
            t, ch = int(r["sample"]) / SAMPLE_RATE, int(r["channel"])
            if events and ch == events[-1][1] and t - events[-1][0] < EVENT_SPAN_S:
                continue
            events.append((t, ch))
        if len(events) >= min_events:
            conns.append(_connection_from_events(int(grp[0]["access_addr"]), int(grp[0]["crc_init"]), events, len(grp)))
    conns.sort(key=lambda c: (c["t_first"], c["access_addr"]))
    return conns


def discover_coded_connections(rx, captures: np.ndarray, min_events: int = 4, offset_hz=None):
    """LE Coded PHY connections found from their empty coded PDUs alone, without an AUX_CONNECT_REQ (include/btle_b200.h,
    "Coded connection discovery").  captures: int8 [40, n_int8]; rows 0..36 are scanned in one rx.discover_coded() call
    (offset_hz: a scalar or one per capture of the 40, passed for rows 0..36 when given).  The candidates are grouped
    exactly as discover_connections() groups its own.  Each dict carries "coded": True, `tracked` False and no hop or
    interval (None): coded connections use CSA#2, which neither the hop inference nor the 1M walk follows."""
    captures = np.ascontiguousarray(captures, dtype=np.int8)
    assert captures.shape[0] == 40
    kw = {} if offset_hz is None else {"offset_hz": np.broadcast_to(np.asarray(offset_hz, dtype=np.float32), (40,))[0:37]}
    conns = _group_candidates(rx.discover_coded(captures[0:37], np.arange(37, dtype=np.int32), **kw), min_events)
    for c in conns:
        c.update(coded=True, tracked=False, hop=None, interval=None)
    return conns


def channel_freq_mhz(channel: int) -> int:
    """get_freq_by_channel_number (btle_rx.c:1006-1022), in MHz."""
    if channel == 37:
        return 2402
    if channel == 38:
        return 2426
    if channel == 39:
        return 2480
    if 0 <= channel <= 10:
        return 2404 + 2 * channel
    if 11 <= channel <= 36:
        return 2428 + 2 * (channel - 11)
    raise ValueError("channel number must be within 0~39")


def hop_events(conns) -> list:
    """The NDJSON `hop` events (btle_json.h:21-24) the reference's FSM emits for these connections
    (`btj_emit_hop` call sites btle_rx.c:2420, :2448, :2486, :2520), with sample time as `ts`:
      track_drop   0->0  CONNECT_REQ without a full channel map (:2417-2424), stays on the advertising channel
      track_start  0->1  CONNECT_REQ accepted, first data channel (:2427-2450); for a tracked discovered connection
                         (discover_connections) at t_first on first_channel
    Untracked discovered connections emit nothing.
      chan_change  2->3  hop after an event that had a CRC-ok packet (:2472-2488)
      chan_change  3->3  hop after an event without one, "Hop: skip" (:2504-2522)
    Returns dicts in time order; hop_events_ndjson() formats them."""
    out = []
    for c in conns:
        if c.get("discovered") and not c.get("tracked"):
            continue                             # a channel sequence the follower cannot predict: nothing to emit
        base = {"v": 1, "t": "hop", "aa": f"{c['access_addr']:08x}", "crc_init": f"{c['crc_init'] & 0xFFFFFF:06x}",
                "hop": c["hop"], "chm": c["chm"]}
        if not c.get("tracked"):
            out.append(dict(base, ts=c["t"], event="track_drop", state_from=0, state_to=0, ch=c["adv_channel"], freq_mhz=0,
                            interval_us=0))
            continue
        interval_us = c["interval"] * 1250                                                    # :2430
        if c.get("discovered"):                  # no CONNECT_REQ: tracking starts with the first empty PDU seen
            ts, first_ch = c["t_first"], c["first_channel"]
        else:
            ts, first_ch = c["t"], c["hop"] % 37                                              # :2434
        out.append(dict(base, ts=ts, event="track_start", state_from=0, state_to=1, ch=first_ch,
                        freq_mhz=channel_freq_mhz(first_ch), interval_us=interval_us))
        ev = c.get("events", [])
        for prev, e in zip(ev, ev[1:]):
            out.append(dict(base, ts=e["t_hop"], event="chan_change", state_from=2 if prev["anchored"] else 3, state_to=3,
                            ch=e["channel"], freq_mhz=channel_freq_mhz(e["channel"]), interval_us=interval_us))
    out.sort(key=lambda d: d["ts"])
    return out


def hop_events_ndjson(conns) -> str:
    """One line per event, fields and formats exactly as btj_emit_hop writes them (btle_json.c:132-160)."""
    lines = []
    for d in hop_events(conns):
        lines.append('{"v":1,"t":"hop","ts":%.6f,"event":"%s","state_from":%d,"state_to":%d,"ch":%d,"freq_mhz":%d,'
                     '"aa":"%s","crc_init":"%s","interval_us":%d,"hop":%d,"chm":"%s"}'
                     % (d["ts"], d["event"], d["state_from"], d["state_to"], d["ch"], d["freq_mhz"], d["aa"], d["crc_init"],
                        d["interval_us"], d["hop"], d["chm"]))
    return "\n".join(lines) + ("\n" if lines else "")


# ---- live: every connection on a streaming session (DESIGN.md §6.4) -----------------------------------------------------
class ConnectionMonitor:
    """decode_connections() while the 40 channel captures are still arriving.  `session` is an RxStreams over 40 captures,
    row c = BLE channel c (cfgs 0..39 as make_cfgs(40, channel=range(40))), fed only through this monitor.  It needs the
    session's push, finish, add_cfg, remove_cfg, resident, set_discover and candidates.

    Captures 37..39 keep their advertising cfg; the cfgs of 0..36 are removed and, with discover=True, discovery runs on
    them.  After each hand-out of records, every CONNECT_REQ and every discovered (access address, CRC init) group that
    has reached `min_events` events gets one cfg on each of the 37 data captures, from chunk `resident` on: the two sets
    still on the device are decoded with it too (backfill).  A discovered group whose access address a CONNECT_REQ
    announced is skipped, as in decode_connections().  Grouping is incremental with discover_connections()' rules; once
    the captures have ended it gives the same connections.  Each connection carries `from_chunk` (its traffic starts
    there: for a discovered connection, traffic before the set in front of the one in which it reached min_events is not
    decoded) and `traffic`, in time order.  idle_s: a connection with no CRC-ok packet for that long stops being decoded
    (`until_chunk`); None keeps every connection to the end, as decode_connections() does.  group_s: a candidate group
    that has not reached min_events and has had no event for that long is forgotten, so that noise groups do not pile up
    over a long session (the default, 8 s, is twice the longest connection interval; a group paused longer than that
    starts again, where discover_connections() would continue it).  offset_hz (a scalar or one per capture): the
    session's carrier-offset correction of each capture (RxStreams.set_offset), from the first set on.  symbol_spaced:
    the connection cfgs carry BTLE_CFG_SYMBOL_SPACED; the session must have been opened with cfgs that carry it (a
    session has one discriminator mode).  lowpass, offset_search: likewise BTLE_CFG_LOWPASS, BTLE_CFG_OFFSET_SEARCH.  centre_hits / correct: the connection cfgs
    carry BTLE_CFG_CENTRE_HITS / BTLE_CFG_CORRECT (per cfg, so the session's own cfgs may carry them or not).  Discovery
    keeps its own rule."""

    N_CAPTURES = 40

    def __init__(self, session, min_events: int = 4, idle_s: float | None = None, discover: bool = True, group_s: float = 8.0,
                 offset_hz=None, symbol_spaced: bool = False, centre_hits: bool = False, correct: bool = False, lowpass: bool = False,
                 offset_search: bool = False):
        self.session, self.min_events, self.idle_s, self.group_s = session, int(min_events), idle_s, group_s
        self._symbol_spaced, self._centre_hits, self._correct = bool(symbol_spaced), bool(centre_hits), bool(correct)
        self._lowpass, self._offset_search = bool(lowpass), bool(offset_search)
        if offset_hz is not None:
            for c, hz in enumerate(np.broadcast_to(np.asarray(offset_hz, dtype=np.float32), (self.N_CAPTURES,))):
                session.set_offset(c, float(hz))
        for c in range(37):
            session.remove_cfg(c)
        if discover:
            session.set_discover(list(range(37)) + [-1] * 3)
        self._adv = []
        self._creq, self._disc = [], {}          # CONNECT_REQ connections in arrival order; (aa, crc) -> discovered one
        self._groups = {}                        # (aa, crc) -> [events [(t, channel)], n_candidates]
        self._owner = {}                         # stable cfg index -> connection
        self._t_now = 0.0

    # ---- feeding ----
    def push(self, capture: int, iq) -> np.ndarray:
        """session.push(); returns the records handed out (advertising and connection cfgs alike)."""
        recs = self.session.push(capture, iq)
        self._hand_out(recs)
        return recs

    def finish(self) -> np.ndarray:
        """session.finish(), repeated while connections found in the last records still get their backfill."""
        out = []
        while True:
            recs = self.session.finish()
            out.append(recs)
            if not self._hand_out(recs):
                return np.concatenate(out)

    # ---- results ----
    @property
    def adv(self) -> np.ndarray:
        """Advertising records handed out so far (stream = capture 37..39)."""
        from ._native import REC_DTYPE
        return np.concatenate(self._adv) if self._adv else np.zeros(0, dtype=REC_DTYPE)

    def connections(self) -> list:
        """decode_connections()' list so far: CONNECT_REQ connections in (advertising capture, time) order, then the
        discovered ones by (t_first, access address); each with `from_chunk` and `traffic` (stream = channel)."""
        creq = sorted(self._creq, key=lambda c: (c["adv_channel"], c["t"]))
        disc = sorted((c for c in self._disc.values() if not c.get("_dropped")), key=lambda c: (c["t_first"], c["access_addr"]))
        out = []
        for c in creq + disc:
            d = {k: v for k, v in c.items() if not k.startswith("_")}
            d["traffic"] = self._traffic(c)
            out.append(d)
        return out

    @staticmethod
    def _traffic(c):
        tr = np.concatenate(c["_traffic"])
        t = tr["chunk"].astype(np.int64) * 8192 + tr["n0"]
        tr = tr[np.lexsort((tr["channel"], t))].copy()
        tr["stream"] = tr["channel"]
        return tr

    # ---- one hand-out ----
    def _start(self, c, t_start):
        s = self.session
        frm = s.resident
        c["from_chunk"], c["_cfgs"], c["_last_ok"] = frm, [], t_start
        from ._native import REC_DTYPE
        c["_traffic"] = [np.zeros(0, dtype=REC_DTYPE)]
        for ch in range(37):
            j, _ = s.add_cfg(ch, frm, channel=ch, access_addr=c["access_addr"], access_mask=0xFFFFFFFF, crc_init=c["crc_init"], raw=0, rssi=0,
                           symbol_spaced=self._symbol_spaced, centre_hits=self._centre_hits, correct=self._correct,
                           lowpass=self._lowpass, offset_search=self._offset_search)
            c["_cfgs"].append(j)
            self._owner[j] = c
        return 37

    def _stop(self, c):
        for j in c.pop("_cfgs", []):
            c["until_chunk"] = self.session.remove_cfg(j)

    def _hand_out(self, recs) -> int:
        """Records (and the candidates of the same sets) -> connections; returns the number of cfgs added."""
        added = 0
        if len(recs):
            self._t_now = max(self._t_now, float((recs["chunk"].astype(np.int64) * 8192 + recs["n0"]).max()) / SAMPLE_RATE)
        adv = recs[(recs["stream"] >= 37) & (recs["stream"] < self.N_CAPTURES)]
        if len(adv):
            self._adv.append(adv.copy())
        for r in adv:
            c = parse_connect_req(r)
            if c is None:
                continue
            c["tracked"] = c["chm"] == "1fffffffff" and c["interval"] > 0
            self._creq.append(c)
            for d in self._disc.values():        # announced after all: the CONNECT_REQ connection takes it over
                if d["access_addr"] == c["access_addr"] and not d.get("_dropped"):
                    d["_dropped"] = True
                    self._stop(d)
            added += self._start(c, c["t"])
        mine = recs[recs["stream"] >= self.N_CAPTURES]
        if len(mine):
            order = np.argsort(mine["stream"], kind="stable")
            mine = mine[order]
            cuts = np.flatnonzero(np.diff(mine["stream"])) + 1
            for part in np.split(mine, cuts):
                c = self._owner[int(part[0]["stream"])]
                c["_traffic"].append(part.copy())
                ok = part[part["crc_bad"] == 0]
                if len(ok):
                    c["_last_ok"] = max(c["_last_ok"], float((ok["chunk"].astype(np.int64) * 8192 + ok["n0"]).max()) / SAMPLE_RATE)
        added += self._discover()
        if self.idle_s is not None:
            for c in self._creq + list(self._disc.values()):
                if c.get("_cfgs") and self._t_now - c["_last_ok"] > self.idle_s:
                    self._stop(c)
        return added

    def _discover(self) -> int:
        cand = self.session.candidates()
        changed = set()                          # groups with new events: only those can start or change a connection
        if len(cand):
            self._t_now = max(self._t_now, float(cand["sample"].max()) / SAMPLE_RATE)
            # the sets' candidates all lie behind the previous hand-out's: grouping them in sample order continues the
            # batch rule of discover_connections()
            cand = cand[np.lexsort((cand["sample"], cand["crc_init"], cand["access_addr"]))]
            key = cand["access_addr"].astype(np.int64) << 24 | cand["crc_init"].astype(np.int64)
            for grp in np.split(cand, np.flatnonzero(np.diff(key)) + 1):
                key_ = (int(grp[0]["access_addr"]), int(grp[0]["crc_init"]))
                g = self._groups.setdefault(key_, [[], 0])
                changed.add(key_)
                events = g[0]
                for r in grp:
                    t, ch = int(r["sample"]) / SAMPLE_RATE, int(r["channel"])
                    if events and ch == events[-1][1] and t - events[-1][0] < EVENT_SPAN_S:
                        continue
                    events.append((t, ch))
                g[1] += len(grp)
        if changed:
            for key in [k for k, (ev, _) in self._groups.items() if len(ev) < self.min_events and self._t_now - ev[-1][0] > self.group_s]:
                del self._groups[key]
        added = 0
        announced = {c["access_addr"] for c in self._creq}
        for aa, crc in sorted(changed):
            if (aa, crc) not in self._groups:
                continue
            events, n_cand = self._groups[(aa, crc)]
            if len(events) < self.min_events or aa in announced:
                continue
            c = _connection_from_events(aa, crc, events, n_cand)
            d = self._disc.get((aa, crc))
            if d is None:
                self._disc[(aa, crc)] = c
                added += self._start(c, c["t_first"])
            else:
                d.update(c)
        return added
