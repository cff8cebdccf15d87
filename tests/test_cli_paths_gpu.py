"""btle_rx_b200's raw captures all go through one streaming session: its print order (sample time, but each capture's
records in the capture's own, reference order) and its stop rule (SIGINT prints only what a full run prints first)."""
import json
import os
import re
import signal
import subprocess
import time

import numpy as np
import pytest

import orc
from btle_b200 import synth
from btle_b200.rx import BtleRx
from test_cli import CLI, _normalise_text, run

MASK = 0x0F000000          # 4 access-address bits: noise gives hits everywhere, some of them out of time order


@pytest.fixture(scope="module", autouse=True)
def built():
    import __graft_entry__ as ge
    ge.build()
    assert os.path.exists(CLI)


@pytest.fixture(scope="module")
def noise(tmp_path_factory):
    """Two noise captures (8 chunks and the look-ahead); the first one's records, from BtleRx.rx_batch, contain a record
    that starts before the record in front of it: a hit at n0 < 0 of chunk k+1 behind a late one of chunk k."""
    d = tmp_path_factory.mktemp("noise")
    caps = [np.random.default_rng(seed).integers(-128, 128, 8 * 16384 + 3008, dtype=np.int8) for seed in (0, 1)]
    for name, iq in zip(("a.bin", "b.bin"), caps):
        iq.tofile(d / name)
    rec = BtleRx(0).rx(caps[0], channel=37, access_mask=MASK, raw=1)
    t = rec["chunk"].astype(np.int64) * 8192 + rec["n0"]
    assert np.any(np.diff(t) < 0)
    return d, rec


def _raw_lines_by_channel(out):
    """-r lines ("sec.usec PktN ChC AA:... Raw:...") of each channel, without the run-wide packet number."""
    by = {}
    for l in out.splitlines():
        m = re.match(r"^(\d+\.\d+) Pkt\d+ Ch(\d+) (.*)$", l)
        if m:
            by.setdefault(int(m.group(2)), []).append(f"{m.group(1)} {m.group(3)}")
    return by


@pytest.mark.gpu
@pytest.mark.skipif(not orc.ref_available(), reason="oracle/_ref not built")
def test_cli_out_of_time_order_record_keeps_the_reference_order(noise):
    d, rec = noise
    p = run(["-i", str(d / "a.bin"), "-c", "37", "-m", f"{MASK:x}", "-r"])
    assert p.returncode == 0, p.stdout + p.stderr
    q = subprocess.run([orc.REF_DRIVER, "sinks", str(d / "a.bin"), "37", "8e89bed6", "555555", f"{MASK:x}", "1", "0", "0", "0",
                        "-", "-", "-"], capture_output=True, text=True, check=True)
    mine = _normalise_text(p.stdout)
    assert len(mine) == len(rec) and mine == _normalise_text(q.stdout)


@pytest.mark.gpu
def test_cli_multi_capture_prints_each_capture_as_its_single_run(noise):
    """With a second capture on another channel, the lines of each channel (times included) are those of that capture's
    own run: the out-of-order record is not moved in front of its predecessor."""
    d, rec = noise
    multi = run(["-i", f"{d}/a.bin:37", "-i", f"{d}/b.bin:9", "-m", f"{MASK:x}", "-r"])
    assert multi.returncode == 0, multi.stdout + multi.stderr
    got = _raw_lines_by_channel(multi.stdout)
    for name, ch in (("a.bin", 37), ("b.bin", 9)):
        single = run(["-i", str(d / name), "-c", str(ch), "-m", f"{MASK:x}", "-r"])
        assert single.returncode == 0
        assert got[ch] == _raw_lines_by_channel(single.stdout)[ch], ch
    assert len(got[37]) == len(rec) and len(got[9]) > 20


@pytest.mark.gpu
def test_cli_sigint_prints_a_prefix_of_the_full_run(tmp_path):
    """A capture piped into -i - and stopped by SIGINT part way: exit 0 with a 'stop' status, and the packets printed are
    the first ones of the full run (no record of a chunk whose look-ahead had not arrived)."""
    iq, _ = synth.make_adv_stream(64 * 16384, seed=43, channel=37, slot_samples=3000)
    raw = iq.numpy().tobytes()
    f = tmp_path / "iq.bin"
    f.write_bytes(raw)
    args = ["-c", "37", "-j", "-Q", "--segment-chunks", "8"]
    pk = lambda lines: [l for l in lines if '"t":"pkt"' in l]
    full = run(["-i", str(f)] + args)
    assert full.returncode == 0
    full_pk = pk(full.stdout.splitlines())
    p = subprocess.Popen([CLI, "-i", "-"] + args, stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    p.stdin.write(raw[:40 * 16384 + 1000])             # 39 chunks with their look-ahead, and a part of the 40th
    p.stdin.flush()
    lines = []
    t0 = time.time()
    while time.time() - t0 < 60 and len(pk(lines)) < 20:   # packets of the completed segment sets, while the pipe is open
        lines.append(p.stdout.readline().decode().rstrip("\n"))
    assert len(pk(lines)) >= 20
    p.send_signal(signal.SIGINT)
    try:
        p.stdin.close()
    except BrokenPipeError:
        pass
    lines += p.stdout.read().decode().splitlines()
    assert p.wait(timeout=30) == 0
    assert json.loads(lines[-1])["event"] == "stop"
    got = pk(lines)
    assert 20 <= len(got) < len(full_pk) and got == full_pk[:len(got)]
