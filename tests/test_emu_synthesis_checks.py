"""One matrix of invalid inputs through every synthesis entry point and world_b200_modify_batch, on the single-thread
host emulation (CPU).  Every call is rejected before anything is queued: EINVAL, no kernel launched, no output written,
last_error from this call starting with the entry point's family ("Synthesis:" or "modify:") and naming the bad
utterance where there is one, and the context works afterwards.  The context runs at the smallest scratch budget, so
the host calls cut the batch into chunks of two utterances and the bad one (the last) lies in a later chunk."""
import ctypes as C
import re

import numpy as np
import pytest

from test_stage_paths import SMALL_BUDGET, _with_budget
from world_b200.api import _ptr

EINVAL = 3
FS, FP, FFT, DIMS = 16000, 5.0, 1024, 40
BINS = FFT // 2 + 1
Y = 2 * FS                  # 2 s rows: about 24 MB of scratch per utterance, two per pass at the smallest budget
L = 401
N = 4
SHORT_F, SHORT_Y = 41, 1600   # the valid call after the errors: short utterances in the same rows

# family: (entry point, who, coded rows, takes nbit, takes factors)
FAMILIES = {
    "synthesis_batch": ("world_b200_synthesis_batch", "Synthesis", False, False, False),
    "synthesis_coded_batch": ("world_b200_synthesis_coded_batch", "Synthesis", True, False, False),
    "synthesis_coded_batch_pcm16": ("world_b200_synthesis_coded_batch_pcm16", "Synthesis", True, False, False),
    "synthesis_coded_batch_modified": ("world_b200_synthesis_coded_batch_modified", "Synthesis", True, True, True),
    "synthesis_coded_host": ("world_b200_synthesis_coded_host", "Synthesis", True, True, False),
    "synthesis_coded_host_modified": ("world_b200_synthesis_coded_host_modified", "Synthesis", True, True, True),
    "modify_batch": ("world_b200_modify_batch", "modify", False, False, True),
}


class Rows:
    """f0, full and coded envelope rows of N utterances, and sentinel outputs."""

    def __init__(self, world):
        k = np.arange(BINS) / BINS
        self.f0 = np.full((N, L), 150.0)
        self.sp = np.ascontiguousarray(np.broadcast_to(np.exp(-6.0 * k) * 1e-3, (N, L, BINS)))
        self.ap = np.full((N, L, BINS), 0.3)
        self.csp = np.ascontiguousarray(world.code_spectral_envelope(self.sp, FS, FFT, DIMS))
        self.cap = np.ascontiguousarray(world.code_aperiodicity(self.ap, FS, FFT))
        world.synchronize()
        self.f0_0, self.sp_0 = self.f0.copy(), self.sp.copy()
        self.y = np.full((N, Y), -7.0)
        self.y16 = np.full((N, Y), -7, dtype=np.int16)

    def untouched(self):
        return ((self.y == -7.0).all() and (self.y16 == -7).all() and np.array_equal(self.f0, self.f0_0)
                and np.array_equal(self.sp, self.sp_0))


def call(world, rows, family, f0=True, sp=True, ap=True, y=True, n=N, fs=FS, fp=FP, fft=FFT, dims=DIMS, nbit=None,
         f0_lengths=None, y_lengths=None, f0_scale=None):
    entry, _, coded, takes_nbit, _ = FAMILIES[family]
    fn = getattr(world.lib, entry)
    fl = (C.c_int * N)(*(f0_lengths or [L] * N))
    yl = (C.c_int * N)(*(y_lengths or [Y] * N))
    pcm16 = family.endswith("pcm16") or nbit == 16
    yp = _ptr(rows.y16 if pcm16 else rows.y) if y else None
    f0p = _ptr(rows.f0) if f0 else None
    scale = (C.c_double * N)(*(f0_scale or [1.2] * N))
    if family == "modify_batch":
        return fn(world._h, f0p, fl, n, L, _ptr(rows.sp) if sp else None, fft, fs, scale, (C.c_double * N)(*[0.9] * N))
    if not coded:
        return fn(world._h, f0p, fl, n, L, _ptr(rows.sp) if sp else None, _ptr(rows.ap) if ap else None, fft, fp, fs,
                  yl, Y, yp)
    head = (world._h, f0p, fl, n, L, _ptr(rows.csp) if sp else None, dims, _ptr(rows.cap) if ap else None, fft, fp,
            fs, yl, Y)
    if family.endswith("modified"):
        return fn(*head, scale, (C.c_double * N)(*[0.9] * N), nbit or 0, yp)
    if takes_nbit:
        return fn(*head, nbit or 0, yp)
    return fn(*head, yp)


def cases(family):
    _, _, coded, takes_nbit, factors = FAMILIES[family]
    last = N - 1
    bad_scale = [1.2] * (N - 1) + [-1.0]
    # (what, keyword arguments of call(), text the message contains besides the family)
    if family == "modify_batch":
        return [
            ("f0 NULL", dict(f0=False), "f0_scale"),
            ("spectrogram NULL", dict(sp=False), "spectral_ratio"),
            ("fs 0", dict(fs=0), "fs"),
            ("n_utts -1", dict(n=-1), "n_utts"),
            ("fft_size 1000", dict(fft=1000), "fft_size"),
            ("f0 length beyond its row", dict(f0_lengths=[L] * (N - 1) + [L + 1]), f"f0_lengths[{last}]"),
            ("bad factor", dict(f0_scale=bad_scale), f"f0_scale[{last}]"),
        ]
    out = [
        ("f0 NULL", dict(f0=False), "must be given"),
        ("rows NULL", dict(sp=False), "must be given"),
        ("y NULL", dict(y=False), "must be given"),
        ("fs 0", dict(fs=0), "fs"),
        ("frame_period 0", dict(fp=0.0), "frame_period"),
        ("n_utts -1", dict(n=-1), "n_utts"),
        ("fft_size 1000", dict(fft=1000), "fft_size"),
        ("f0 length 1", dict(f0_lengths=[L] * (N - 1) + [1]), f"f0_lengths[{last}]"),
        ("y length beyond its row", dict(y_lengths=[Y] * (N - 1) + [Y + 1]), f"y_lengths[{last}]"),
    ]
    if not coded:
        out.append(("aperiodicity NULL", dict(ap=False), "must be given"))
    if takes_nbit:
        out.append(("nbit 8", dict(nbit=8), "nbit"))
    if coded:
        out.append(("dims 0", dict(dims=0), "number_of_dimensions"))
        out.append(("coded aperiodicity NULL at 16 kHz", dict(ap=False), "coded_aperiodicity"))
    if factors:
        out.append(("bad factor", dict(f0_scale=bad_scale), f"f0_scale[{last}]"))
    return out


@pytest.fixture(scope="module")
def small(emu):
    w = _with_budget(emu, SMALL_BUDGET)
    yield w
    w.close()


@pytest.mark.parametrize("family", list(FAMILIES))
def test_emu_synthesis_rejects_before_queuing(small, family):
    lib, h = small.lib, small._h
    rows = Rows(small)
    who = FAMILIES[family][1]
    pcm = np.zeros(16, dtype=np.int16)
    out = np.zeros(16)
    for what, kw, named in cases(family):
        # a different failing call just before: the case's last_error must be its own
        assert lib.world_b200_pcm_to_double_batch(h, _ptr(pcm), 12, 1, 16, None, _ptr(out)) == EINVAL
        stale = lib.world_b200_last_error(h).decode()
        before = small.launch_count()
        rc = call(small, rows, family, **kw)
        err = lib.world_b200_last_error(h).decode()
        assert rc == EINVAL, f"{family}, {what}: returned {rc}"
        assert small.launch_count() == before, f"{family}, {what}: kernels were launched"
        assert rows.untouched(), f"{family}, {what}: an output was written"
        assert err != stale and err.startswith(who + ":"), f"{family}, {what}: last_error {err!r}"
        assert named in err, f"{family}, {what}: last_error {err!r} does not name {named!r}"
    # the context works afterwards (short utterances in the same rows, so the run stays quick)
    before = small.launch_count()
    rc = call(small, rows, family, f0_lengths=[SHORT_F] * N, y_lengths=[SHORT_Y] * N)
    small.synchronize()
    assert rc == 0, f"{family}: the context does not work after the errors: {lib.world_b200_last_error(h).decode()}"
    assert small.launch_count() > before
    if family == "modify_batch":
        assert not np.array_equal(rows.f0, rows.f0_0)
    else:
        assert not rows.untouched(), f"{family}: the valid call wrote nothing"


def test_emu_synthesis_host_chunks_at_small_budget(small, capfd, monkeypatch):
    """The rows above run in chunks of two utterances at the smallest budget: the last utterance is in a later chunk
    than the first, so the host calls' rejections above happen before any chunk is queued."""
    rows = Rows(small)
    monkeypatch.setenv("WB_HOST_TRACE", "1")
    capfd.readouterr()
    # every utterance at its full length: the sizes decide the chunks, not the contents
    assert call(small, rows, "synthesis_coded_host", nbit=16) == 0
    found = re.findall(r"\[wb trace\] synthesis chunk (\d+) chunks (\d+)", capfd.readouterr().err)
    assert found and found[-1] == ("2", "2"), found
