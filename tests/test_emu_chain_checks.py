"""One matrix of invalid inputs through every analysis chain family and voice transformation, device and host, on the
single-thread host emulation (CPU).  Every call is rejected before anything is queued: EINVAL, no kernel launched, no
output written, last_error from this call naming the bad utterance, and the context works afterwards.  The host
pipelines run with one-utterance sub-chunks and two-utterance chunks, so the bad utterance (the last) lies in a later
chunk than the first."""
import ctypes as C

import numpy as np
import pytest

import dio_ranges_common as dr
import f0_ranges_common as hr
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST, CheapTrickOption, D4COption, _ptr

EINVAL = 3
DIMS = 24
FS = 16000
LENS = [2400, 2800, 3200, 4000]   # the last utterance is the longest: f0_stride one frame short names it alone
STRIDE = 4000

# family: (entry point without its option suffix, which also prefixes its errors; coded rows)
FAMILIES = {
    "analyze_batch": ("analyze_batch", False),
    "analyze_coded_batch": ("analyze_coded_batch", True),
    "analyze_host": ("analyze_host", False),
    "analyze_coded_host": ("analyze_coded_host", True),
    "analyze_coded_batch spectral": ("analyze_coded_batch", True),
    "analyze_coded_host spectral": ("analyze_coded_host", True),
    "transform_batch": ("transform_batch", False),
    "transform_host": ("transform_host", False),
}


def _x():
    rng = np.random.default_rng(7)
    t = np.arange(STRIDE) / FS
    x = 0.3 * np.sin(2 * np.pi * 180.0 * t)[None, :] + 0.05 * rng.standard_normal((len(LENS), STRIDE))
    for u, m in enumerate(LENS):
        x[u, m:] = 0.0
    return np.ascontiguousarray(x)


class Chain:
    """One family's entry points on fixed inputs, with outputs that start as a sentinel."""

    def __init__(self, world, family):
        self.world, self.lib, self.family = world, world.lib, family
        self.entry, self.coded = FAMILIES[family]
        self.spectral = family.endswith("spectral")
        self.transform = self.entry.startswith("transform")
        self.x = _x()
        n = len(LENS)
        self.L = max(world.frames(FS, m) for m in LENS)
        if self.transform:
            self.Y = max(world.transform_samples(FS, m, 5.0) for m in LENS)
            shapes = [(n, self.Y)]
        else:
            bins = world.cheaptrick_option(FS).fft_size // 2 + 1
            widths = (DIMS, max(1, world.number_of_aperiodicities(FS))) if self.coded else (bins, bins)
            shapes = [(n, self.L), (n, self.L), (n, self.L, widths[0]), (n, self.L, widths[1])]
        self.outs = [np.full(s, -7.0) for s in shapes]

    def call(self, method=F0_DIO_STONEMASK, nbit=0, lens=LENS, f0_stride=None, ho=None, do=None, dims=DIMS, ct=None,
             opt=None, fs=FS):
        n = len(LENS)
        ao = opt or self.world.analysis_option(fs, method)
        head = (self.world._h, _ptr(self.x)) + ((nbit,) if self.coded or self.transform else ()) + (
            n, STRIDE, (C.c_int * n)(*lens), fs, C.byref(ao))
        if self.transform:
            return getattr(self.lib, f"world_b200_{self.entry}")(*head, ho, do, None, None, None, 0,
                                                                 _ptr(self.outs[0]), self.Y, None)
        outs = (_ptr(self.outs[0]), _ptr(self.outs[1]), self.L if f0_stride is None else f0_stride,
                _ptr(self.outs[2]), _ptr(self.outs[3]))
        if self.coded:
            outs = (dims,) + outs
        if self.spectral:
            cts = [self.world.cheaptrick_option(fs) for _ in LENS]
            if ct is not None:
                cts[-1].fft_size = ct
            ct_arr = (CheapTrickOption * n)(*cts)
            d4_arr = (D4COption * n)(*[self.world.d4c_option() for _ in LENS])
            return getattr(self.lib, f"world_b200_{self.entry}_spectral_options")(*head, ho, do, ct_arr, d4_arr, *outs)
        if ho is not None:
            return getattr(self.lib, f"world_b200_{self.entry}_options")(*head, ho, *outs)
        if do is not None:
            return getattr(self.lib, f"world_b200_{self.entry}_dio_options")(*head, do, *outs)
        return getattr(self.lib, f"world_b200_{self.entry}")(*head, *outs)


def _cases(ch):
    n = len(LENS)
    hopts = (hr.HarvestOption * n)(*hr.options([(71.0, 800.0)] * n))
    dopts = (dr.DioOption * n)(*dr.options([(71.0, 800.0, 2.0, 0.1)] * n))
    bad_fp = hr.options([(71.0, 800.0)] * n)
    bad_fp[3].frame_period = 1.0
    bad_fp = (hr.HarvestOption * n)(*bad_fp)
    bad_range = hr.options([(71.0, 800.0)] * n)
    bad_range[3].f0_floor = -5.0
    bad_range = (hr.HarvestOption * n)(*bad_range)
    fmax = ch.world.cheaptrick_option(FS).fft_size // 4 + 1
    # (what, call, text the message contains)
    cases = [
        ("length beyond its row in a later chunk", lambda: ch.call(lens=LENS[:3] + [STRIDE + 1]), "x_lengths[3]"),
        ("length 0", lambda: ch.call(lens=LENS[:2] + [0, LENS[3]]), "x_lengths[2]"),
        ("DIO options on a Harvest chain", lambda: ch.call(method=F0_HARVEST, do=dopts), "f0_method"),
        ("Harvest options on a DIO chain", lambda: ch.call(ho=hopts), "f0_method"),
        ("frame_period differs", lambda: ch.call(method=F0_HARVEST, ho=bad_fp), "utterance 3)"),
        ("F0 range below zero", lambda: ch.call(method=F0_HARVEST, ho=bad_range), "utterance 3)"),
        # the stages' sampling-rate limits: StoneMask's window at 96 kHz, D4C's transforms at 192 kHz
        ("DIO chain at 96 kHz", lambda: ch.call(fs=96000), "StoneMask: sampling rate"),
        ("Harvest chain at 192 kHz", lambda: ch.call(method=F0_HARVEST, fs=192000), "D4C: sampling rate"),
    ]
    if ch.coded or ch.transform:
        cases.append(("nbit 12", lambda: ch.call(nbit=12), "nbit"))
    if not ch.transform:
        cases.append(("f0_stride too small", lambda: ch.call(f0_stride=ch.L - 1), "utterance 3)"))
    if ch.coded:
        cases.append(("dims 0", lambda: ch.call(dims=0), "number_of_dimensions"))
        cases.append(("dims fft/4 + 2", lambda: ch.call(dims=fmax + 1), "number_of_dimensions"))
    if ch.spectral:
        cases.append(("CheapTrick fft_size 1000", lambda: ch.call(ct=1000), "utterance 3)"))
    return cases


@pytest.mark.parametrize("family", list(FAMILIES))
def test_emu_chain_rejects_before_queuing(emu, monkeypatch, family):
    monkeypatch.setenv("WB_HOST_CHUNK", "2")
    monkeypatch.setenv("WB_HOST_SUB", "1")
    ch = Chain(emu, family)
    lib, h = emu.lib, emu._h
    other = (C.c_int * 2)(800, 801)
    t = np.zeros(16)
    for what, fn, named in _cases(ch):
        # a different failing call just before: the case's last_error must be its own
        assert lib.world_b200_cheaptrick_batch(h, _ptr(ch.x), 2, 800, other, FS, _ptr(t), _ptr(t), None, 11,
                                               C.byref(emu.cheaptrick_option(FS)), _ptr(np.zeros(16 * 513))) == EINVAL
        stale = lib.world_b200_last_error(h).decode()
        before = emu.launch_count()
        rc = fn()
        err = lib.world_b200_last_error(h).decode()
        assert rc == EINVAL, f"{family}, {what}: returned {rc}"
        assert emu.launch_count() == before, f"{family}, {what}: kernels were launched"
        for o in ch.outs:
            assert (o == -7.0).all(), f"{family}, {what}: an output was written"
        assert err != stale and err.startswith(ch.entry + ":"), f"{family}, {what}: last_error {err!r}"
        assert named in err, f"{family}, {what}: last_error {err!r} does not name {named!r}"
    assert ch.call() == 0, f"{family}: the context does not work after the errors"
    assert not (ch.outs[-1] == -7.0).all(), f"{family}: the valid call wrote nothing"
