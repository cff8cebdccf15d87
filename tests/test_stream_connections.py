"""hop.ConnectionMonitor without a GPU: the monitor on a fake session that follows the streaming session's contract
(btle_b200_streams_add_cfg / remove_cfg / resident / set_discover / take_cands) with the oracle.  At every set size its
incremental grouping equals discover_connections(), and its connections and traffic equal decode_connections()'."""
import numpy as np
import pytest

import discover_ref as R
import orc
from btle_b200._native import CAND_DTYPE, REC_DTYPE
from btle_b200.hop import ConnectionMonitor, decode_connections, discover_connections
from btle_b200.rx import make_cfgs
from test_rx_multi import OracleMultiRx, connections_capture

CHUNK = 16384
LOOK = 4096


class FakeSession:
    """The session's contract on whole captures known in advance: set k = chunks [k*seg, (k+1)*seg) is submitted once
    every capture has seg chunks + 4096 bytes of it, and handed out when set k+1 is submitted (or at finish).  A cfg's
    records are the oracle's on its whole capture, kept for [from, until); an added cfg is decoded over the two most
    recent sets (backfill), handed out with the set when it is still in flight, else by the next push / finish."""

    def __init__(self, captures, seg):
        self.caps, self.seg = captures, seg
        self.n_int8 = captures.shape[1]
        self.nchunks = self.n_int8 // CHUNK
        base = make_cfgs(40, channel=list(range(40)))
        self.entries = [[i, base[i:i + 1], 0, 1 << 40] for i in range(40)]
        self.fill = [0] * 40
        self.submitted = []            # [(first chunk, n chunks, [live cfg indices])]
        self.handed = 0                # sets handed out
        self.waiting = []              # backfill records for the next push / finish
        self.disc = [-1] * 40
        self.scan_from = {}            # set -> channels scanned
        self.cands = []
        self._recs, self._all_cands = {}, None
        self.finished = False
        self.jobs = {}                 # set -> cfgs added while it was in flight

    def _records(self, j):
        cap, cfg, _, _ = self.entries[j]
        key = (cap, cfg.tobytes())
        if key not in self._recs:
            c = cfg[0]
            self._recs[key] = orc.rx_flags(self.caps[cap], int(c["rssi"]), channel=int(c["channel"]), access_addr=int(c["access_addr"]),
                                           access_mask=int(c["access_mask"]), crc_init=int(c["crc_init"]), raw=int(c["raw"]), stream=0)
        return self._recs[key]

    def _decode(self, j, lo, hi):
        _, _, frm, until = self.entries[j]
        r = self._records(j)
        r = r[(r["chunk"] >= max(lo, frm)) & (r["chunk"] < min(hi, until))].copy()
        r["stream"] = j
        return r

    def _hand_out(self, k, jobs):
        lo, nch, live, last = self.submitted[k]
        out = [self._decode(j, lo, lo + nch) for j in sorted(set(live) | set(jobs.get(k, [])))]
        if k in self.scan_from:
            if self._all_cands is None:
                self._all_cands = R.discover_batch(self.caps[0:37], np.arange(37))
            c = self._all_cands
            s0, s1 = lo * 8192, (1 << 60) if last else (lo + nch) * 8192
            self.cands.append(c[(c["sample"] >= s0) & (c["sample"] < s1)])
        return out

    def _submit(self, nch, last=False):
        lo = sum(s[1] for s in self.submitted)
        live = [j for j, e in enumerate(self.entries) if e[2] < lo + nch and e[3] > lo]
        self.submitted.append((lo, nch, live, last))
        if any(c >= 0 for c in self.disc):
            self.scan_from[len(self.submitted) - 1] = True

    def push(self, capture, iq):
        self.fill[capture] += np.asarray(iq).size
        out, self.waiting = self.waiting, []
        while all(f >= (len(self.submitted) + 1) * self.seg * CHUNK + LOOK for f in self.fill):
            self._submit(self.seg)
            k = len(self.submitted) - 2
            if k >= 0:
                out += self._hand_out(k, self.jobs)
                self.handed = k + 1
        return np.concatenate(out) if out else np.zeros(0, dtype=REC_DTYPE)

    def finish(self):
        out, self.waiting = self.waiting, []
        if not self.finished:
            self.finished = True
            lo = sum(s[1] for s in self.submitted)
            tail = self.nchunks - lo
            for k in range(self.handed, len(self.submitted)):
                out += self._hand_out(k, self.jobs)
            self._submit(tail, last=True)
            out += self._hand_out(len(self.submitted) - 1, self.jobs)
            self.handed = len(self.submitted)
        return np.concatenate(out) if out else np.zeros(0, dtype=REC_DTYPE)

    @property
    def resident(self):
        if not self.submitted:
            return 0
        return self.submitted[max(0, len(self.submitted) - 2)][0]

    def add_cfg(self, capture, from_chunk=None, **fields):
        frm = self.resident if from_chunk is None else from_chunk
        assert frm >= self.resident
        j = len(self.entries)
        self.entries.append([capture, make_cfgs(1, **fields), frm, 1 << 40])
        for k in range(max(0, len(self.submitted) - 2), len(self.submitted)):
            if k < self.handed:        # already handed out: by the next push / finish
                self.waiting.append(self._decode(j, self.submitted[k][0], self.submitted[k][0] + self.submitted[k][1]))
            else:                      # in flight: with its set
                self.jobs.setdefault(k, []).append(j)
        return j, frm

    def remove_cfg(self, index):
        e = self.entries[index]
        e[3] = max(e[2], sum(s[1] for s in self.submitted))
        return e[3]

    def set_discover(self, channels):
        self.disc = list(channels)

    def candidates(self):
        out = np.concatenate(self.cands) if self.cands else np.zeros(0, dtype=CAND_DTYPE)
        self.cands = []
        return out


KEYS = ("access_addr", "crc_init", "tracked", "interval", "hop", "t_first", "first_channel", "n_events", "n_candidates")


@pytest.fixture(scope="module")
def offline():
    cap, _ = connections_capture()
    return cap, decode_connections(OracleMultiRx(), cap), discover_connections(R.OracleDiscoverRx(), cap)


@pytest.mark.parametrize("seg", [3, 8, 16, 40])
def test_monitor_on_oracle_session_equals_offline(offline, seg):
    cap, (adv, conns), found = offline
    mon = ConnectionMonitor(FakeSession(cap, seg))
    rng = np.random.default_rng(seg)
    pos = [0] * 40
    while any(p < cap.shape[1] for p in pos):
        i = int(rng.integers(40))
        n = int(rng.choice([5000, CHUNK, 4 * CHUNK]))
        mon.push(i, cap[i, pos[i]:pos[i] + n])
        pos[i] += n
    mon.finish()
    # the incremental grouping: every group with enough events is one of discover_connections()'
    groups = {k: v for k, v in mon._groups.items() if len(v[0]) >= mon.min_events}
    assert sorted(groups) == sorted((c["access_addr"], c["crc_init"]) for c in found)
    for c in found:
        events, n_cand = groups[(c["access_addr"], c["crc_init"])]
        assert len(events) == c["n_events"] and n_cand == c["n_candidates"] and events[0] == (c["t_first"], c["first_channel"])
    live = mon.connections()
    assert len(live) == len(conns) == 3
    for a, b in zip(live, conns):
        assert {k: a.get(k) for k in KEYS} == {k: b.get(k) for k in KEYS}
        want = b["traffic"][b["traffic"]["chunk"] >= a["from_chunk"]]
        assert a["traffic"].tobytes() == want.tobytes() and len(want) > 5
        if not b.get("discovered"):
            assert a["from_chunk"] == 0 and a["traffic"].tobytes() == b["traffic"].tobytes()
