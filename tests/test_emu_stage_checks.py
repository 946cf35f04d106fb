"""One matrix of invalid inputs through the nine CheapTrick, D4C and StoneMask stage entry points, on the single-thread
host emulation (CPU).  Every call is rejected before anything is queued: EINVAL, no kernel launched, no output
written, last_error from this call starting with the stage's name ("CheapTrick:", "D4C:" or "StoneMask:") and naming
the bad utterance where one is at fault, and the context works afterwards.  The single-option forms follow the rules of
the per-utterance forms: a non-finite q1 or threshold is refused by both."""
import ctypes as C

import numpy as np
import pytest

from world_b200.api import CheapTrickOption, D4COption, _ptr

EINVAL = 3
FS, FFT, DIMS = 16000, 1024, 24
BINS = FFT // 2 + 1
N, STRIDE = 4, 1600
LAST = N - 1

# entry point: (stage, coded rows, one option per utterance)
ENTRIES = {
    "world_b200_cheaptrick_batch": ("CheapTrick", False, False),
    "world_b200_cheaptrick_coded_batch": ("CheapTrick", True, False),
    "world_b200_cheaptrick_batch_options": ("CheapTrick", False, True),
    "world_b200_cheaptrick_coded_batch_options": ("CheapTrick", True, True),
    "world_b200_d4c_batch": ("D4C", False, False),
    "world_b200_d4c_coded_batch": ("D4C", True, False),
    "world_b200_d4c_batch_options": ("D4C", False, True),
    "world_b200_d4c_coded_batch_options": ("D4C", True, True),
    "world_b200_stonemask_batch": ("StoneMask", False, False),
}


class Rows:
    """x, time axis and f0 of N utterances, and an output that starts as a sentinel."""

    def __init__(self, world, entry):
        stage, coded, _ = ENTRIES[entry]
        self.L = world.frames(FS, STRIDE)
        t = np.arange(STRIDE) / FS
        self.x = np.ascontiguousarray(np.broadcast_to(0.3 * np.sin(2 * np.pi * 150.0 * t), (N, STRIDE)))
        self.t = np.ascontiguousarray(np.broadcast_to(np.arange(self.L) * 0.005, (N, self.L)))
        self.f0 = np.full((N, self.L), 150.0)
        width = () if stage == "StoneMask" else (DIMS if stage == "CheapTrick" else 1,) if coded else (BINS,)
        self.out = np.full((N, self.L) + width, -7.0)

    def untouched(self):
        return (self.out == -7.0).all() and (self.f0 == 150.0).all()


def call(world, rows, entry, x=True, t=True, f0=True, out=True, opts=True, n=N, fs=FS, x_lengths=None,
         f0_lengths=None, fft=FFT, q=None, row=BINS, dims=DIMS):
    """fft / q (q1 or threshold): the one option's, or the last utterance's in the per-utterance forms."""
    stage, coded, per_utt = ENTRIES[entry]
    head = (world._h, _ptr(rows.x) if x else None, n, STRIDE, (C.c_int * N)(*(x_lengths or [STRIDE] * N)), fs,
            _ptr(rows.t) if t else None, _ptr(rows.f0) if f0 else None,
            (C.c_int * N)(*(f0_lengths or [rows.L] * N)), rows.L)
    dst = _ptr(rows.out) if out else None
    fn = getattr(world.lib, entry)
    if stage == "StoneMask":
        return fn(*head, dst)
    if stage == "CheapTrick":
        o = [world.cheaptrick_option(FS) for _ in range(N)]
        o[-1].fft_size = fft
        if q is not None:
            o[-1].q1 = q
        opt = ((CheapTrickOption * N)(*o) if per_utt else C.byref(o[-1])) if opts else None
        tail = (dims,) if coded else (row,) if per_utt else ()
        return fn(*head, opt, *tail, dst)
    o = [world.d4c_option() for _ in range(N)]
    if q is not None:
        o[-1].threshold = q
    if per_utt:
        sizes = (C.c_int * N)(*([FFT] * (N - 1) + [fft]))
        return fn(*head, sizes, (D4COption * N)(*o) if opts else None, *(() if coded else (row,)), dst)
    return fn(*head, fft, C.byref(o[-1]) if opts else None, dst)


def cases(entry):
    """(what, keyword arguments of call(), texts the message contains besides the stage's name)"""
    stage, coded, per_utt = ENTRIES[entry]
    named = (f"(utterance {LAST})",) if per_utt else ()
    out = [
        ("x NULL", dict(x=False), ("must be given",)),
        ("time_axis NULL", dict(t=False), ("must be given",)),
        ("f0 NULL", dict(f0=False), ("must be given",)),
        ("output NULL", dict(out=False), ("must be given",)),
        ("n_utts -1", dict(n=-1), ("n_utts",)),
        ("fs 0", dict(fs=0), ("fs",)),
        ("x length 0", dict(x_lengths=[STRIDE] * LAST + [0]), (f"x_lengths[{LAST}]", f"(utterance {LAST})")),
        ("x length beyond its row", dict(x_lengths=[STRIDE] * LAST + [STRIDE + 1]),
         (f"x_lengths[{LAST}]", f"(utterance {LAST})")),
        ("f0 length beyond its row", dict(f0_lengths=[1] * LAST + [10 ** 6]), (f"f0_lengths[{LAST}]", f"(utterance {LAST})")),
    ]
    if stage == "StoneMask":
        out.append(("96 kHz", dict(fs=96000), ("sampling rate",)))
        return out
    out.append(("options NULL", dict(opts=False), ("must be given",)))
    if stage == "CheapTrick":
        out += [
            ("fft_size 1000", dict(fft=1000), ("power of two",) + named),
            ("fft_size 16384", dict(fft=16384), ("power of two",) + named),
            ("q1 NaN", dict(q=float("nan")), ("q1",) + named),
        ]
        if coded:
            out += [("dims 0", dict(dims=0), ("number_of_dimensions",)),
                    ("dims fft/4 + 2", dict(dims=FFT // 4 + 2), ("number_of_dimensions",))]
    else:
        out += [
            ("fft_size 3", dict(fft=3), ("at least 4",) + named),
            ("threshold inf", dict(q=float("inf")), ("threshold",) + named),
            ("192 kHz", dict(fs=192000), ("sampling rate",)),
        ]
    if per_utt and not coded:
        out.append(("row_stride one short", dict(row=BINS - 1), ("row_stride",)))
    return out


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_emu_stage_rejects_before_queuing(emu, entry):
    lib, h = emu.lib, emu._h
    rows = Rows(emu, entry)
    stage = ENTRIES[entry][0]
    pcm = np.zeros(16, dtype=np.int16)
    tmp = np.zeros(16)
    for what, kw, texts in cases(entry):
        # a different failing call just before: the case's last_error must be its own
        assert lib.world_b200_pcm_to_double_batch(h, _ptr(pcm), 12, 1, 16, None, _ptr(tmp)) == EINVAL
        stale = lib.world_b200_last_error(h).decode()
        before = emu.launch_count()
        rc = call(emu, rows, entry, **kw)
        err = lib.world_b200_last_error(h).decode()
        assert rc == EINVAL, f"{entry}, {what}: returned {rc}"
        assert emu.launch_count() == before, f"{entry}, {what}: kernels were launched"
        assert rows.untouched(), f"{entry}, {what}: an output was written"
        assert err != stale and err.startswith(stage + ":"), f"{entry}, {what}: last_error {err!r}"
        for text in texts:
            assert text in err, f"{entry}, {what}: last_error {err!r} does not name {text!r}"
    # the context works afterwards
    before = emu.launch_count()
    rc = call(emu, rows, entry)
    emu.synchronize()
    assert rc == 0, f"{entry}: the context does not work after the errors: {lib.world_b200_last_error(h).decode()}"
    assert emu.launch_count() > before
    assert not rows.untouched(), f"{entry}: the valid call wrote nothing"
