"""Checks of the voice transformation (world_b200_transform_batch / world_b200_transform_host): PCM in, analysis,
F0 scaling and formant shift, synthesis at a per-utterance frame period, PCM out.  The same assertions run against the
host emulation (CPU) and the CUDA library (-m gpu).

The oracle is the stepwise chain of the same library: analyze_batch (full rows, the same options) -> modify ->
synthesis with frame_period * time_scale[u], grouped by time_scale, and the pcm16 rule for 16-bit output.  The call
must equal it bit for bit.  The reference's demo program and its Synthesis at a scaled frame period hold the chain to
the reference."""
import ctypes as C
import os

import numpy as np

import modify_common as mc
import test_parity_common as pc
from test_stage_paths import SMALL_BUDGET, _with_budget
from world_b200.api import F0_DIO_STONEMASK, F0_HARVEST

EINVAL = 3
METHODS = {"harvest": F0_HARVEST, "dio": F0_DIO_STONEMASK}
TIME_SCALES = (0.8, 1.0, 1.25, 2.0)


# ---- inputs -----------------------------------------------------------------------------------------------------------
def pcm_rows(x, nbit):
    """Host rows of x (float64 in [-1, 1)) as the call takes them: float64 for nbit 0, int16 for 16, else uint8 rows of
    nbit/8 little-endian bytes per sample."""
    if nbit == 0:
        return np.ascontiguousarray(x, dtype=np.float64)
    scale = float(1 << (nbit - 1))
    v = np.clip(np.round(x * scale), -scale, scale - 1).astype(np.int64)
    if nbit == 16:
        return v.astype(np.int16)
    b = (v.astype("<i4").view(np.uint8)).reshape(x.shape[0], x.shape[1], 4)[:, :, :nbit // 8]
    return np.ascontiguousarray(b.reshape(x.shape[0], -1))


def high_tone(fs, n, hz=750.0):
    """A steady harmonic tone at hz: scaled by 2 it asks for more than the 1,200 pulses per second (plus 64) Synthesis
    first lays its arrays out for when it is the pass's longest output, so its pass is laid out again from the counts."""
    t = np.arange(n) / fs
    x = sum(0.3 / k * np.sin(2 * np.pi * k * hz * t) for k in range(1, int(4000.0 / hz) + 1))
    return x + 0.003 * np.random.default_rng(7).uniform(-1, 1, n)


def batch(fs, seconds, seeds, with_tone=True):
    """A ragged batch of synthetic speech (tests/synth.py), after the high tone as its first, longest utterance:
    (x, lengths)."""
    from synth import synth_batch
    n = int(seconds * fs)
    x = synth_batch(list(seeds), fs, n).numpy()
    if with_tone:
        x = np.concatenate([high_tone(fs, n)[None], x], axis=0)
    lens = [n - (u * n) // 8 for u in range(x.shape[0])]
    for u, m in enumerate(lens):
        x[u, m:] = 0.0
    return x, lens


def option(world, fs, method, fft=None):
    ao = world.analysis_option(fs, METHODS[method])
    if fft is not None and fft != ao.cheaptrick.fft_size:
        ao.cheaptrick.fft_size = fft
        ao.cheaptrick.f0_floor = max(ao.cheaptrick.f0_floor, 3.0 * fs / (fft - 3.0) + 1.0)
    return ao


def frame_period(ao):
    return ao.dio.frame_period if ao.f0_method == F0_DIO_STONEMASK else ao.harvest.frame_period


def _list(v, n):
    if v is None:
        return None
    return [float(v)] * n if isinstance(v, (int, float)) else [float(t) for t in v]


# ---- the oracle -------------------------------------------------------------------------------------------------------
def stepwise(world, pcm, nbit, fs, ao, lens, scales=None, ratios=None, tscales=None, harvest_options=None,
             dio_options=None, nbit_out=0, f0_out=None):
    """analyze_batch -> modify -> synthesis (one call per distinct time_scale) of the same library; host rows out, 0
    past each length, quantised by the pcm16 rule for nbit_out 16.  f0_out: a list that receives the modified f0."""
    n = pcm.shape[0]
    P = pc.make(world, pcm, dtype=pcm.dtype)
    X = world.pcm_to_double(P, nbit, lens) if nbit else P
    t, f0, sp, ap, fl = world.analyze_batch(X, fs, ao, x_lengths=lens, harvest_options=harvest_options,
                                            dio_options=dio_options)
    fft = ao.cheaptrick.fft_size
    if scales is not None or ratios is not None:
        world.modify(f0, sp, fs, fft, f0_scale=scales, spectral_ratio=ratios, f0_lengths=fl)
    world.synchronize()
    if f0_out is not None:
        f0_out.append(pc.to_np(f0))
    fp = frame_period(ao)
    ts = _list(tscales, n) or [1.0] * n
    yl = [world.transform_samples(fs, lens[u], fp, ts[u]) for u in range(n)]
    y = np.zeros((n, max(yl)))
    for s in sorted(set(ts)):
        idx = [u for u in range(n) if ts[u] == s]
        Y = max(yl[u] for u in idx)
        ys = world.synthesis(f0[idx], sp[idx], ap[idx], fft, fp * s, fs, Y, f0_lengths=[fl[u] for u in idx],
                             y_lengths=[yl[u] for u in idx])
        world.synchronize()
        ys = pc.to_np(ys)
        for i, u in enumerate(idx):
            y[u, :yl[u]] = ys[i, :yl[u]]
    if nbit_out == 16:
        y = mc.quantised(y)
        for u in range(n):
            y[u, yl[u]:] = 0
    return y, yl


def transform(world, pcm, nbit, fs, ao, lens, scales=None, ratios=None, tscales=None, harvest_options=None,
              dio_options=None, nbit_out=0):
    y, yl = world.transform(pc.make(world, pcm, dtype=pcm.dtype), nbit, fs, ao, f0_scale=scales,
                            spectral_ratio=ratios, time_scale=tscales, x_lengths=lens, harvest_options=harvest_options,
                            dio_options=dio_options, dtype="int16" if nbit_out == 16 else None)
    world.synchronize()
    return pc.to_np(y), yl


# ---- checks -----------------------------------------------------------------------------------------------------------
def check_stepwise(world, fs, fft, method, nbit, seconds=0.6):
    """A ragged batch with a different pitch, formant and tempo factor per utterance (the high tone scaled by 2.0 takes
    the relaid pulse pass; the ratio 2 / fft keeps only bin 0), float64 and 16-bit output, equal to the stepwise
    chain bit for bit."""
    x, lens = batch(fs, seconds, (501, 502, 503, 504))
    pcm = pcm_rows(x, nbit)
    ao = option(world, fs, method, fft)
    n = x.shape[0]
    scales = [2.0, 0.5, 1.3, 0.8, 1.0]
    ratios = [1.1, 1.2, 2.0 / fft, 0.85, 1.0]
    tscales = [2.0, 0.8, 1.0, 1.25, 1.0]
    assert len(scales) == n and set(tscales) == set(TIME_SCALES)
    f0s = []
    want, yl = stepwise(world, pcm, nbit, fs, ao, lens, scales, ratios, tscales, f0_out=f0s)
    assert (f0s[0][0] > 1200.0).sum() > 10, "the scaled tone does not ask for the relaid pulse pass"
    for u in range(n):
        assert np.abs(want[u, :yl[u]]).max() > 1e-3, f"utterance {u} is silent"
    got, gl = transform(world, pcm, nbit, fs, ao, lens, scales, ratios, tscales)
    assert gl == yl and got.shape == want.shape
    for u in range(n):
        assert np.array_equal(got[u], want[u]), f"utterance {u} (time_scale {tscales[u]}) differs from the stepwise chain"
    got16, _ = transform(world, pcm, nbit, fs, ao, lens, scales, ratios, tscales, nbit_out=16)
    assert got16.dtype == np.int16
    assert np.array_equal(got16, mc.quantised(want)), "pcm16 differs from the quantised stepwise chain"


def check_relaid_pass(world):
    """The high tone scaled by 2.0 makes synthesis lay its pass out again: one more time-base launch than at 1.0."""
    fs = 16000
    x, lens = batch(fs, 0.5, (511,))
    ao = option(world, fs, "harvest")
    counts = []
    for s in (1.0, 2.0):
        before = world.launch_count()
        transform(world, x, 0, fs, ao, lens, scales=[s, 1.0])
        counts.append(world.launch_count() - before)
    assert counts[1] == counts[0] + 1, f"launches {counts}: the pass was not laid out again"


def check_null_factors(world, fs=16000):
    """All three factor arrays NULL: analyze -> synthesis with no modify step.  Each factor alone equals its chain."""
    x, lens = batch(fs, 0.5, (521, 522), with_tone=False)
    pcm = pcm_rows(x, 16)
    ao = option(world, fs, "harvest")
    want, yl = stepwise(world, pcm, 16, fs, ao, lens)
    got, gl = transform(world, pcm, 16, fs, ao, lens)
    assert gl == yl and np.array_equal(got, want)
    assert yl == [world.transform_samples(fs, m, 5.0) for m in lens]
    for kw in ({"scales": [1.4, 0.6]}, {"ratios": [0.9, 1.15]}, {"tscales": [1.25, 0.8]}):
        want, _ = stepwise(world, pcm, 16, fs, ao, lens, **kw)
        got, _ = transform(world, pcm, 16, fs, ao, lens, **kw)
        assert np.array_equal(got, want), f"{kw}: differs from the stepwise chain"


def check_per_utterance_options(world, method, fs=16000):
    """One F0 option per utterance (Harvest or DIO), equal to the stepwise chain with the same options."""
    x, lens = batch(fs, 0.5, (531, 532, 533))
    ao = option(world, fs, method)
    n = x.shape[0]
    floors, ceils = [200.0, 60.0, 90.0, 71.0], [900.0, 500.0, 400.0, 800.0]
    if method == "harvest":
        opts = [world.harvest_option() for _ in range(n)]
    else:
        opts = [world.dio_option() for _ in range(n)]
    for u, o in enumerate(opts):
        o.f0_floor, o.f0_ceil = floors[u], ceils[u]
    kw = {"harvest_options": opts} if method == "harvest" else {"dio_options": opts}
    scales, ratios, tscales = [1.2, 0.9, 1.0, 1.1], [1.0, 1.1, 0.9, 1.0], [1.0, 1.25, 0.8, 1.0]
    want, _ = stepwise(world, x, 0, fs, ao, lens, scales, ratios, tscales, **kw)
    got, _ = transform(world, x, 0, fs, ao, lens, scales, ratios, tscales, **kw)
    assert np.array_equal(got, want), f"per-utterance {method} options: differs from the stepwise chain"
    plain, _ = transform(world, x, 0, fs, ao, lens, scales, ratios, tscales)
    assert not np.array_equal(plain, got), "the per-utterance options changed nothing"


def check_small_budget(world, fs=16000, seconds=1.0, n_utts=5, fft=4096, one_per_slice=False):
    """At the smallest scratch budget the batch runs in many slices (one utterance each where one_per_slice) and gives
    the default context's result bit for bit."""
    from synth import synth_batch
    n = int(seconds * fs)
    x = synth_batch(list(range(541, 541 + n_utts)), fs, n).numpy()
    lens = [n - 997 * u for u in range(n_utts)]
    ao = option(world, fs, "dio", fft)
    pcm = pcm_rows(x, 16)
    args = ([1.1, 0.9, 1.0, 1.3, 0.7][:n_utts], [1.0, 1.2, 0.8, 1.0, 1.1][:n_utts], [1.0, 2.0, 0.8, 1.25, 1.0][:n_utts])
    frames = world.frames(fs, n, 5.0)
    rows = n * 8 + frames * 16 + frames * (fft // 2 + 1) * 16
    lanes = 1 if world.xp == "numpy" else 2
    per_slice = max(1, int(SMALL_BUDGET / lanes / 2 // rows))
    assert per_slice < n_utts / 2 and (per_slice == 1 or not one_per_slice), f"{per_slice} utterances per slice"
    small = _with_budget(world, SMALL_BUDGET)
    try:
        outs, launches = [], []
        for w in (world, small):
            before = w.launch_count()
            outs.append(transform(w, pcm, 16, fs, ao, lens, *args, nbit_out=16)[0])
            launches.append(w.launch_count() - before)
    finally:
        small.close()
    assert launches[1] > launches[0], f"launches: {launches[0]} by default, {launches[1]} at the small budget"
    assert np.array_equal(outs[0], outs[1]), "the sliced result differs"
    want, _ = stepwise(world, pcm, 16, fs, ao, lens, *args, nbit_out=16)
    assert np.array_equal(outs[0], want), "differs from the stepwise chain"


def check_host_equals_device(world, pinned=False, fs=22050):
    """transform_host equals transform bit for bit, float64 and 16-bit out, in one chunk and in chunks of two
    utterances; whole rows come back, 0 past each length."""
    x, lens = batch(fs, 0.5, (551, 552, 553, 554))
    pcm = pcm_rows(x, 16)
    ao = option(world, fs, "harvest")
    n = x.shape[0]
    kw = dict(scales=[1.2, 0.8, 1.0, 1.5, 0.9], ratios=[1.1, 0.9, 1.0, 1.2, 0.95], tscales=[1.0, 2.0, 0.8, 1.25, 1.0])
    old = os.environ.get("WB_HOST_CHUNK")
    try:
        for nbit_out in (0, 16):
            want, yl = transform(world, pcm, 16, fs, ao, lens, nbit_out=nbit_out, **kw)
            dt = np.int16 if nbit_out == 16 else np.float64
            for chunk in (None, "2"):
                if chunk:
                    os.environ["WB_HOST_CHUNK"] = chunk
                else:
                    os.environ.pop("WB_HOST_CHUNK", None)
                xin, out = pcm, np.full(want.shape, 7, dtype=dt)
                if pinned:
                    import torch
                    xin = torch.from_numpy(pcm).pin_memory()
                    out = torch.full(want.shape, 7, dtype=torch.int16 if nbit_out == 16 else torch.float64).pin_memory()
                got, gl = world.transform_host(xin, 16, fs, ao, f0_scale=kw["scales"], spectral_ratio=kw["ratios"],
                                               time_scale=kw["tscales"], x_lengths=lens,
                                               dtype="int16" if nbit_out == 16 else None, out=out)
                got = pc.to_np(got)
                assert gl == yl
                for u in range(n):
                    assert (got[u, yl[u]:] == 0).all(), f"utterance {u}: samples past its length are not 0"
                assert np.array_equal(got, want), f"nbit_out {nbit_out}, chunk {chunk}: host differs from device"
    finally:
        if old is None:
            os.environ.pop("WB_HOST_CHUNK", None)
        else:
            os.environ["WB_HOST_CHUNK"] = old


def check_invalid(world):
    """Every bad argument is EINVAL before any work: nothing is launched, y keeps its sentinel, and last_error names the
    first bad utterance.  n_utts 0 returns 0."""
    fs, n = 16000, 4
    x, lens = batch(fs, 0.3, (561, 562, 563), with_tone=True)
    pcm = pcm_rows(x, 16)
    X = pc.make(world, pcm, dtype=np.int16)
    stride = pcm.shape[1]
    ao = option(world, fs, "harvest")
    yl = [world.transform_samples(fs, m, 5.0) for m in lens]
    Y = max(yl)
    y = pc.make(world, np.full((n, Y), -7.0))
    lib = world.lib
    good = [1.0] * n

    def bad(u, v):
        vals = list(good)
        vals[u] = v
        vals[3] = v
        return vals

    def d(v):
        return None if v is None else (C.c_double * len(v))(*v)

    def call(nbit=16, xl=lens, opt=ao, ho=None, do=None, sc=None, ra=None, ts=None, nbit_out=0, y_stride=Y, count=n,
             host=False):
        fn = lib.world_b200_transform_host if host else lib.world_b200_transform_batch
        xp = pcm.ctypes.data if host else cs_ptr(X)
        yp = yh.ctypes.data if host else cs_ptr(y)
        return lambda: fn(world._h, xp, nbit, count, stride, (C.c_int * n)(*xl), fs, C.byref(opt), ho, do, d(sc),
                          d(ra), d(ts), nbit_out, yp, y_stride, None)

    def opt_with(**kv):
        o = option(world, fs, "harvest")
        for k, v in kv.items():
            sub, field = k.split("__")
            setattr(getattr(o, sub), field, v)
        return o

    yh = np.full((n, Y), -7.0)
    hopts = (type(world.harvest_option()) * n)(*[world.harvest_option() for _ in range(n)])
    hopts[2].frame_period = 2.5
    dopts = (type(world.dio_option()) * n)(*[world.dio_option() for _ in range(n)])
    tiny = float(np.nextafter(2.0 / 1024, 0.0))
    cases = [
        ("nbit 12", call(nbit=12), "nbit"),
        ("nbit_out 8", call(nbit_out=8), "nbit_out"),
        ("nbit_out 32", call(nbit_out=32), "nbit_out"),
        ("x length beyond its row", call(xl=[lens[0], stride + 1, lens[2], lens[3]]), "x_lengths[1]"),
        ("x length 0", call(xl=[lens[0], lens[1], 0, lens[3]]), "x_lengths[2]"),
        ("fft_size 8192", call(opt=opt_with(cheaptrick__fft_size=8192)), "fft_size"),
        ("fft_size 1000", call(opt=opt_with(cheaptrick__fft_size=1000)), "fft_size"),
        ("y_stride below a y_length", call(y_stride=yl[0] - 1), "utterance 0"),
        ("harvest options: frame_period differs", call(ho=hopts), "utterance 2"),
        ("dio options with Harvest", call(do=dopts), "f0_method"),
        ("spectral_ratio c == 0", call(ra=bad(1, tiny)), "spectral_ratio[1]"),
        ("host: time_scale -1", call(ts=bad(2, -1.0), host=True), "time_scale[2]"),
    ]
    for what, v in (("0", 0.0), ("-1", -1.0), ("NaN", float("nan")), ("inf", float("inf"))):
        cases.append((f"time_scale {what}", call(ts=bad(2, v)), "time_scale[2]"))
        cases.append((f"f0_scale {what}", call(sc=bad(1, v)), "f0_scale[1]"))
        cases.append((f"spectral_ratio {what}", call(ra=bad(0, v)), "spectral_ratio[0]"))
    for what, fn, named in cases:
        world._use_current_stream()
        before = world.launch_count()
        rc = fn()
        world.synchronize()
        err = lib.world_b200_last_error(world._h).decode()
        assert rc == EINVAL, f"{what}: returned {rc}"
        assert world.launch_count() == before, f"{what}: kernels were launched"
        assert named in err, f"{what}: last_error {err!r} does not name {named}"
        assert (pc.to_np(y) == -7.0).all() and (yh == -7.0).all(), f"{what}: y was written"
    for host in (False, True):
        rc = call(count=0, host=host)()
        assert rc == 0, f"n_utts 0 ({'host' if host else 'device'}) returned {rc}"
    assert world.transform_samples(fs, 16000, 5.0, float("nan")) == 0
    rc = call(ts=[1.0, 0.8, 0.8, 1.25])()
    world.synchronize()
    assert rc == 0 and not (pc.to_np(y) == -7.0).all(), "the context does not work after the errors"


def cs_ptr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def check_time_scale_vs_reference(world, ref, golden):
    """Synthesis of the fixture's parameters at frame period 5.0 * s, the step transform() adds to the chain, against the
    reference's Synthesis at the same frame period: within 1e-9 of the waveform peak (the bound of every Synthesis
    test)."""
    fs, fft = int(golden["fs"]), int(golden["fft_size"])
    f0, sp, ap = golden["f0_stonemask"], golden["sp"], golden["ap"]
    n = len(golden["pcm"])
    for s in (0.8, 1.25, 2.0):
        y_len = world.transform_samples(fs, n, 5.0, s)
        assert y_len == int((len(f0) - 1) * (5.0 * s) / 1000.0 * fs) + 1
        y = world.synthesis(pc.make(world, f0[None]), pc.make(world, sp[None]), pc.make(world, ap[None]), fft, 5.0 * s,
                            fs, y_len)
        world.synchronize()
        yr = ref.synthesis(f0, sp, ap, fft, 5.0 * s, fs, y_len)
        e = np.abs(pc.to_np(y)[0] - yr).max() / np.abs(yr).max()
        assert e <= 1e-9, f"time_scale {s}: {e:.2e} of the peak"


def check_ref_demo(world, golden, d):
    """The reference's demo program on the fixture against transform_host (16-bit in and out) with the demo's options:
    within 1 LSB, the bound the stepwise chain is held to."""
    fs = int(golden["fs"])
    pcm = np.ascontiguousarray(golden["pcm"].astype(np.int16)[None])
    ao = world.analysis_option(fs, F0_HARVEST)
    ao.harvest.f0_floor, ao.harvest.frame_period, ao.d4c.threshold = 40.0, 5.0, 0.85
    for shift, ratio in ((1.5, 0.85), (0.7, 1.3)):
        want = mc.run_ref_demo(golden, d, shift, ratio)
        got, yl = world.transform_host(pcm, 16, fs, ao, f0_scale=shift, spectral_ratio=ratio, dtype="int16")
        got = np.asarray(got)[0].astype(np.int64)
        assert got.shape == want.shape and yl[0] == len(want)
        assert np.abs(want).max() > 1000
        diff = int(np.abs(got - want).max())
        assert diff <= 1, f"shift {shift} ratio {ratio}: {diff} LSB from the reference demo"
