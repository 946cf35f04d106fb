"""Checks of the coded chain on device arrays (world_b200_analyze_coded_batch and its *_options / *_allgather variants);
the same assertions run against the host emulation (CPU) and the CUDA library (-m gpu)."""
import ctypes as C
import os

import numpy as np
import pytest

import dio_ranges_common as dr
import f0_ranges_common as hr
import test_parity_common as pc
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST, WorldError

EINVAL = 3
DIMS = 24


def pcm_rows(x, nbit):
    """float rows in [-1, 1) -> (rows of nbit-bit little-endian PCM as analyze_coded_* take them, the doubles they
    decode to).  nbit 0 gives the 16-bit doubles themselves."""
    bits = nbit or 16
    q = np.clip(np.round(x * (1 << (bits - 1))), -(1 << (bits - 1)), (1 << (bits - 1)) - 1).astype(np.int64)
    xd = q.astype(np.float64) / float(1 << (bits - 1))
    if nbit == 0:
        return np.ascontiguousarray(xd), xd
    if nbit == 16:
        return np.ascontiguousarray(q.astype(np.int16)), xd
    nb = nbit // 8
    u = (q & ((1 << nbit) - 1)).astype(np.uint64)
    raw = np.zeros((x.shape[0], x.shape[1] * nb), dtype=np.uint8)
    for j in range(nb):
        raw[:, j::nb] = ((u >> np.uint64(8 * j)) & np.uint64(255)).astype(np.uint8)
    return raw, xd


class lane_slices:
    """WB_LANE_SLICES for the duration of a with-block (None: the library's default)."""

    def __init__(self, n):
        self.n, self.saved = n, None

    def __enter__(self):
        self.saved = os.environ.get("WB_LANE_SLICES")
        if self.n is None:
            os.environ.pop("WB_LANE_SLICES", None)
        else:
            os.environ["WB_LANE_SLICES"] = str(self.n)

    def __exit__(self, *exc):
        if self.saved is None:
            os.environ.pop("WB_LANE_SLICES", None)
        else:
            os.environ["WB_LANE_SLICES"] = self.saved


def coded_batch(world, rows, nbit, fs, ao, dims=DIMS, lens=None, slices=None, **kw):
    with lane_slices(slices):
        out = world.analyze_coded_batch(pc.make(world, rows, dtype=rows.dtype), nbit, fs, ao, dims, x_lengths=lens, **kw)
    world.synchronize()
    return [pc.to_np(a) for a in out[:4]] + [out[4]]


def assert_equal_rows(got, want, what):
    for name, g, w in zip(("time_axis", "f0", "coded sp", "coded ap"), got[:4], want[:4]):
        assert g.shape == w.shape, f"{what}: {name} shape {g.shape} vs {w.shape}"
        assert np.array_equal(g, w), f"{what}: {name} differs"


def check_equals_host(world, f0_method, nbit, fs=16000, n_samples=6000, seeds=(151, 152, 153, 154, 155),
                      slice_counts=(1, 2, 3, 7)):
    """Every output of the device chain equals analyze_coded_host's on the same rows, bit for bit, whatever the slice
    count; a ragged batch, PCM widened on the device or doubles."""
    x, lens = hr.ragged_batch(fs, n_samples, list(seeds))
    rows, _ = pcm_rows(0.9 * x / np.abs(x).max(), nbit)
    ao = world.analysis_option(fs, f0_method)
    want = world.analyze_coded_host(rows, nbit, fs, ao, DIMS, x_lengths=lens)
    assert max(want[4]) > min(want[4])
    for u in range(len(seeds)):
        assert (want[1][u, :want[4][u]] > 0).sum() > 10
    for slices in slice_counts:
        got = coded_batch(world, rows, nbit, fs, ao, lens=lens, slices=slices)
        assert got[4] == want[4]
        assert_equal_rows(got, want, f"f0_method {f0_method} nbit {nbit} slices {slices}")


def check_vs_two_step(world, f0_method, fs=16000, n_samples=6000, seeds=(161, 162, 163, 164)):
    """The coded rows against analyze_batch's full rows coded afterwards (code_spectral_envelope / code_aperiodicity):
    f0 and time axis identical, coded rows within the bound of the fused frame kernels against the two-step path."""
    x, lens = hr.ragged_batch(fs, n_samples, list(seeds))
    rows, xd = pcm_rows(0.9 * x / np.abs(x).max(), 16)
    ao = world.analysis_option(fs, f0_method)
    fft = ao.cheaptrick.fft_size
    got = coded_batch(world, rows, 16, fs, ao, lens=lens)
    t, f0, sp, ap, fl = world.analyze_batch(pc.make(world, xd), fs, ao, x_lengths=lens)
    csp = pc.to_np(world.code_spectral_envelope(sp, fs, fft, DIMS, f0_lengths=fl))
    cap = pc.to_np(world.code_aperiodicity(ap, fs, fft, f0_lengths=fl))
    world.synchronize()
    assert got[4] == fl
    for u in range(len(seeds)):
        L = fl[u]
        assert np.array_equal(got[0][u, :L], pc.to_np(t)[u, :L]) and np.array_equal(got[1][u, :L], pc.to_np(f0)[u, :L])
        pc.assert_close_signed(got[2][u, :L], csp[u, :L], f"coded sp vs two-step, utterance {u}", tol=1e-9)
        pc.assert_close_signed(got[3][u, :L], cap[u, :L], f"coded ap vs two-step, utterance {u}", tol=1e-9)


def per_utt_options(f0_method, n):
    if f0_method == F0_HARVEST:
        return {"harvest_options": hr.options([hr.RANGES[u % len(hr.RANGES)] for u in range(n)])}
    return {"dio_options": dr.options([dr.RANGES[u % len(dr.RANGES)] for u in range(n)])}


def check_options(world, f0_method, fs=16000, n_samples=8000, seeds=(131, 132, 133, 134, 135)):
    """Per-utterance F0 options of either method (the speaker-like ranges of f0_ranges_common / dio_ranges_common, one
    per utterance): the rows of analyze_coded_host with the same options, bit for bit, with the options array split
    between slices; and each utterance's f0 differs from what the batch's one option gives somewhere."""
    x, lens = dr.batch(fs, n_samples, list(seeds))
    rows, _ = pcm_rows(x, 16)
    n = len(seeds)
    ao = world.analysis_option(fs, f0_method)
    kw = per_utt_options(f0_method, n)
    want = world.analyze_coded_host(rows, 16, fs, ao, DIMS, x_lengths=lens, **kw)
    for slices in (1, 3):
        got = coded_batch(world, rows, 16, fs, ao, lens=lens, slices=slices, **kw)
        assert_equal_rows(got, want, f"options, f0_method {f0_method} slices {slices}")
    plain = coded_batch(world, rows, 16, fs, ao, lens=lens)
    assert not np.array_equal(plain[1], want[1]), "the per-utterance options changed nothing"


def _ptr(a):
    if a is None:
        return None
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def check_null_outputs(world, fs_list=(16000, 8000), n_samples=5000, seeds=(171, 172, 173)):
    """NULL coded_spectral_envelope skips CheapTrick, NULL coded_aperiodicity skips D4C; the other outputs are the full
    call's.  Below 12 kHz there are no aperiodicity bands: coded_aperiodicity may be NULL and is never written."""
    for fs in fs_list:
        n = int(n_samples * fs / 16000)
        x, lens = hr.ragged_batch(fs, n, list(seeds))
        rows, _ = pcm_rows(0.9 * x / np.abs(x).max(), 16)
        ao = world.analysis_option(fs, F0_DIO_STONEMASK)
        full = coded_batch(world, rows, 16, fs, ao, lens=lens)
        n_ap = world.number_of_aperiodicities(fs)
        fl = full[4]
        L = max(fl)
        xr = pc.make(world, rows, dtype=rows.dtype)
        for drop_sp, drop_ap in ((True, False), (False, True), (True, True)):
            t, f0 = pc.make(world, np.zeros((3, L))), pc.make(world, np.zeros((3, L)))
            csp = None if drop_sp else pc.make(world, np.zeros((3, L, DIMS)))
            # (frames beyond an utterance's count are not written: zeros, like the full call's arrays)
            cap = None if drop_ap else pc.make(world, np.full((3, L, max(1, n_ap)), 0.0 if n_ap else -7.0))
            world._use_current_stream()
            rc = world.lib.world_b200_analyze_coded_batch(world._h, _ptr(xr), 16, 3, rows.shape[1],
                                                          (C.c_int * 3)(*lens), fs, C.byref(ao), DIMS, _ptr(t),
                                                          _ptr(f0), L, _ptr(csp), _ptr(cap))
            world.synchronize()
            assert rc == 0, world.lib.world_b200_last_error(world._h)
            assert np.array_equal(pc.to_np(t), full[0]) and np.array_equal(pc.to_np(f0), full[1])
            if csp is not None:
                assert np.array_equal(pc.to_np(csp), full[2])
            if cap is not None:
                if n_ap > 0:
                    assert np.array_equal(pc.to_np(cap), full[3])
                else:
                    assert (pc.to_np(cap) == -7.0).all(), "coded aperiodicity written below 12 kHz"
        if n_ap == 0:
            assert not full[3].any()


def check_invalid(world):
    """Bad nbit, bad number_of_dimensions, options of the other F0 method or with another frame_period, and lengths
    outside their rows are EINVAL, and nothing is written (the outputs keep their sentinel); the context keeps
    working."""
    fs = 16000
    x, lens = hr.ragged_batch(fs, fs // 2, [61, 62, 63, 64])
    rows, _ = pcm_rows(0.9 * x / np.abs(x).max(), 16)
    n = rows.shape[0]
    ao_h, ao_d = world.analysis_option(fs, F0_HARVEST), world.analysis_option(fs, F0_DIO_STONEMASK)
    L = max(world.frames(fs, v) for v in lens)
    xr = pc.make(world, rows, dtype=rows.dtype)
    outs = [pc.make(world, np.full(s, -7.0)) for s in ((n, L), (n, L), (n, L, DIMS), (n, L, 1))]

    def call(fn, *mid, nbit=16, dims=DIMS, ao=ao_h, stride=rows.shape[1], ls=lens, f0_stride=L):
        world._use_current_stream()
        rc = fn(world._h, _ptr(xr), nbit, n, stride, (C.c_int * n)(*ls), fs, C.byref(ao), *mid, dims, _ptr(outs[0]),
                _ptr(outs[1]), f0_stride, _ptr(outs[2]), _ptr(outs[3]))
        world.synchronize()
        return rc

    lib = world.lib
    fmax = ao_h.cheaptrick.fft_size // 4 + 1
    hopts = (type(hr.options([(71.0, 800.0)])[0]) * n)(*hr.options([(71.0, 800.0)] * n))
    dopts = (type(dr.options([(71.0, 800.0, 2.0, 0.1)])[0]) * n)(*dr.options([(71.0, 800.0, 2.0, 0.1)] * n))
    bad_fp = hr.options([(71.0, 800.0)] * n)
    bad_fp[2].frame_period = 1.0
    bad_fp = (type(bad_fp[0]) * n)(*bad_fp)
    cases = [
        ("nbit 12", lambda: call(lib.world_b200_analyze_coded_batch, nbit=12)),
        ("nbit -16", lambda: call(lib.world_b200_analyze_coded_batch, nbit=-16)),
        ("dims 0", lambda: call(lib.world_b200_analyze_coded_batch, dims=0)),
        ("dims fft/4 + 2", lambda: call(lib.world_b200_analyze_coded_batch, dims=fmax + 1)),
        ("DIO options on a Harvest chain", lambda: call(lib.world_b200_analyze_coded_batch_dio_options, dopts)),
        ("Harvest options on a DIO chain", lambda: call(lib.world_b200_analyze_coded_batch_options, hopts, ao=ao_d)),
        ("frame_period differs", lambda: call(lib.world_b200_analyze_coded_batch_options, bad_fp)),
        ("NULL options", lambda: call(lib.world_b200_analyze_coded_batch_options, None)),
        ("length beyond the row", lambda: call(lib.world_b200_analyze_coded_batch, ls=[lens[0], rows.shape[1] + 1] + lens[2:])),
        ("f0_stride too small", lambda: call(lib.world_b200_analyze_coded_batch, f0_stride=L - 1)),
        ("allgather without a communicator", lambda: call(lib.world_b200_analyze_coded_batch_allgather)),
    ]
    for what, fn in cases:
        assert fn() == EINVAL, what
        for o in outs:
            assert (pc.to_np(o) == -7.0).all(), f"{what}: an output was written"
    with pytest.raises(ValueError):
        world.analyze_coded_batch(xr, 12, fs, ao_h, DIMS, x_lengths=lens)
    with pytest.raises(WorldError, match="error 3: .*number_of_dimensions"):
        world.analyze_coded_batch(xr, 16, fs, ao_h, fmax + 1, x_lengths=lens)
    got = world.analyze_coded_batch(xr, 16, fs, ao_h, DIMS, x_lengths=lens)
    world.synchronize()
    assert (pc.to_np(got[1])[0, :got[4][0]] > 0).sum() > 10
