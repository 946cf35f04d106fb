"""ctypes mirror of the batched C ABI (include/world_b200.h) and of the reference's operator
names (Dio / Harvest / StoneMask / CheapTrick / D4C, src/world/*.h).

This module is plumbing: it loads ``world_b200/lib/libworld_b200.so`` (hand-written sm_90a CUDA
behind an extern "C" ABI), hands it raw pointers and returns arrays.  There is no Python or CPU
implementation of any stage behind it -- if the library or a CUDA device is missing, loading
or ``World()`` raises.

Arrays: every batched call takes ``x`` as a 2-D float64 array ``[n_utts, x_stride]``.
``torch`` CUDA tensors are passed by device pointer (zero copy, work is enqueued on torch's
current stream); outputs are allocated with torch on the same device.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "lib", "libworld_b200.so")


class DioOption(C.Structure):  # dio.h:16-23
    _fields_ = [("f0_floor", C.c_double), ("f0_ceil", C.c_double), ("channels_in_octave", C.c_double),
                ("frame_period", C.c_double), ("speed", C.c_int), ("allowed_range", C.c_double)]


class HarvestOption(C.Structure):  # harvest.h:16-20
    _fields_ = [("f0_floor", C.c_double), ("f0_ceil", C.c_double), ("frame_period", C.c_double)]


class CheapTrickOption(C.Structure):  # cheaptrick.h:16-20
    _fields_ = [("q1", C.c_double), ("f0_floor", C.c_double), ("fft_size", C.c_int)]


class D4COption(C.Structure):  # d4c.h:16-18
    _fields_ = [("threshold", C.c_double)]


class AnalysisOption(C.Structure):
    _fields_ = [("f0_method", C.c_int), ("dio", DioOption), ("harvest", HarvestOption),
                ("cheaptrick", CheapTrickOption), ("d4c", D4COption)]


F0_DIO_STONEMASK = 0
F0_HARVEST = 1

_P = C.c_void_p
_IP = C.POINTER(C.c_int)

# every symbol include/world_b200.h and include/world/*.h declare: (restype, argtypes)
ABI = {
    "world_b200_create": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "world_b200_destroy": (None, [_P]),
    "world_b200_set_stream": (C.c_int, [_P, _P]),
    "world_b200_set_scratch_budget": (C.c_int, [_P, C.c_ulonglong]),
    "world_b200_synchronize": (C.c_int, [_P]),
    "world_b200_trim": (C.c_int, [_P]),
    "world_b200_last_error": (C.c_char_p, [_P]),
    "world_b200_launch_count": (C.c_ulonglong, [_P]),
    "world_b200_frames": (C.c_int, [C.c_int, C.c_int, C.c_double]),
    "world_b200_randn_stream": (C.c_int, [_P, C.c_uint, _P]),
    "world_b200_randn_window": (C.c_int, [_P, C.c_ulonglong, C.c_uint, _P]),
    "world_b200_rfft_test": (C.c_int, [_P, _P, C.c_int, _P]),
    "world_b200_sfft_test": (C.c_int, [_P, _P, C.c_int, _P]),
    "world_b200_fp64_peak": (C.c_int, [_P, C.POINTER(C.c_double)]),
    "world_b200_fp64_tensor_peak": (C.c_int, [_P, C.POINTER(C.c_double)]),
    "world_b200_profile": (C.c_int, [_P, C.c_int]),
    "world_b200_profile_report": (C.c_int, [_P, C.c_char_p, C.c_ulonglong]),
    "world_b200_dio_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(DioOption), _P, _P, C.c_int]),
    "world_b200_dio_batch_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(DioOption), _P, _P,
                                               C.c_int]),
    "world_b200_harvest_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(HarvestOption), _P, _P, C.c_int]),
    "world_b200_harvest_batch_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(HarvestOption), _P,
                                                   _P, C.c_int]),
    "world_b200_stonemask_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP, C.c_int, _P]),
    "world_b200_cheaptrick_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP, C.c_int,
                                              C.POINTER(CheapTrickOption), _P]),
    "world_b200_d4c_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP, C.c_int, C.c_int,
                                       C.POINTER(D4COption), _P]),
    "world_b200_cheaptrick_coded_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP, C.c_int,
                                                    C.POINTER(CheapTrickOption), C.c_int, _P]),
    "world_b200_d4c_coded_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP, C.c_int, C.c_int,
                                             C.POINTER(D4COption), _P]),
    "world_b200_synthesis_batch": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, _P, C.c_int, C.c_double, C.c_int, _IP,
                                             C.c_int, _P]),
    "world_b200_synthesis_coded_batch": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_double,
                                                   C.c_int, _IP, C.c_int, _P]),
    "world_b200_synthesis_coded_batch_pcm16": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int,
                                                         C.c_double, C.c_int, _IP, C.c_int, _P]),
    "world_b200_synthesis_coded_host": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_double,
                                                  C.c_int, _IP, C.c_int, C.c_int, _P]),
    "world_b200_default_analysis_option": (None, [C.c_int, C.c_int, C.POINTER(AnalysisOption)]),
    "world_b200_analyze_host": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(AnalysisOption),
                                          _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(AnalysisOption),
                                           _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_batch_allgather": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(AnalysisOption),
                                                     _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_host_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(AnalysisOption),
                                                  C.POINTER(HarvestOption), _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_batch_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(AnalysisOption),
                                                   C.POINTER(HarvestOption), _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_batch_allgather_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int,
                                                             C.POINTER(AnalysisOption), C.POINTER(HarvestOption), _P,
                                                             _P, C.c_int, _P, _P]),
    "world_b200_analyze_host_dio_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(AnalysisOption),
                                                      C.POINTER(DioOption), _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_batch_dio_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int,
                                                       C.POINTER(AnalysisOption), C.POINTER(DioOption), _P, _P, C.c_int,
                                                       _P, _P]),
    "world_b200_analyze_batch_allgather_dio_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int,
                                                                 C.POINTER(AnalysisOption), C.POINTER(DioOption), _P,
                                                                 _P, C.c_int, _P, _P]),
    "world_b200_comm_unique_id": (C.c_int, [_P, C.c_int]),
    "world_b200_comm_init": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int]),
    "world_b200_comm_destroy": (C.c_int, [_P]),
    "world_b200_allgather_rows": (C.c_int, [_P, _P, C.c_ulonglong, C.c_ulonglong]),
    # legacy single-utterance API (host pointers)
    "Dio": (None, [_P, C.c_int, C.c_int, C.POINTER(DioOption), _P, _P]),
    "Harvest": (None, [_P, C.c_int, C.c_int, C.POINTER(HarvestOption), _P, _P]),
    "StoneMask": (None, [_P, C.c_int, C.c_int, _P, _P, C.c_int, _P]),
    "CheapTrick": (None, [_P, C.c_int, C.c_int, _P, _P, C.c_int, C.POINTER(CheapTrickOption), _P]),
    "D4C": (None, [_P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, C.POINTER(D4COption), _P]),
    "Synthesis": (None, [_P, C.c_int, _P, _P, C.c_int, C.c_double, C.c_int, C.c_int, _P]),
    "InitializeDioOption": (None, [C.POINTER(DioOption)]),
    "InitializeHarvestOption": (None, [C.POINTER(HarvestOption)]),
    "InitializeCheapTrickOption": (None, [C.c_int, C.POINTER(CheapTrickOption)]),
    "InitializeD4COption": (None, [C.POINTER(D4COption)]),
    "GetSamplesForDIO": (C.c_int, [C.c_int, C.c_int, C.c_double]),
    "GetSamplesForHarvest": (C.c_int, [C.c_int, C.c_int, C.c_double]),
    "GetFFTSizeForCheapTrick": (C.c_int, [C.c_int, C.POINTER(CheapTrickOption)]),
    "GetF0FloorForCheapTrick": (C.c_double, [C.c_int, C.c_int]),
    # codec (row f2) and ingest (row f3)
    "world_b200_code_aperiodicity_batch": (C.c_int, [_P, _P, C.c_int, _IP, C.c_int, C.c_int, C.c_int, _P]),
    "world_b200_decode_aperiodicity_batch": (C.c_int, [_P, _P, C.c_int, _IP, C.c_int, C.c_int, C.c_int, _P]),
    "world_b200_code_spectral_envelope_batch": (C.c_int, [_P, _P, C.c_int, _IP, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "world_b200_decode_spectral_envelope_batch": (C.c_int, [_P, _P, C.c_int, _IP, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "world_b200_wav_parse": (C.c_int, [_P, C.c_ulonglong, _IP, _IP, _IP, C.POINTER(C.c_ulonglong)]),
    "world_b200_pcm_to_double_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, _P]),
    "world_b200_analyze_coded_host": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                C.POINTER(AnalysisOption), C.c_int, _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_coded_host_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                        C.POINTER(AnalysisOption), C.POINTER(HarvestOption), C.c_int,
                                                        _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_coded_host_dio_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                            C.POINTER(AnalysisOption), C.POINTER(DioOption), C.c_int,
                                                            _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_coded_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                 C.POINTER(AnalysisOption), C.c_int, _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_coded_batch_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                         C.POINTER(AnalysisOption), C.POINTER(HarvestOption), C.c_int,
                                                         _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_coded_batch_dio_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                             C.POINTER(AnalysisOption), C.POINTER(DioOption), C.c_int,
                                                             _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_coded_batch_allgather": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                           C.POINTER(AnalysisOption), C.c_int, _P, _P, C.c_int, _P,
                                                           _P]),
    "world_b200_analyze_coded_batch_allgather_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                                   C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                                   C.c_int, _P, _P, C.c_int, _P, _P]),
    "world_b200_analyze_coded_batch_allgather_dio_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP,
                                                                       C.c_int, C.POINTER(AnalysisOption),
                                                                       C.POINTER(DioOption), C.c_int, _P, _P, C.c_int,
                                                                       _P, _P]),
    # host-only file glue (tools/audioio.h, tools/parameterio.h)
    "wavwrite": (None, [_P, C.c_int, C.c_int, C.c_int, C.c_char_p]),
    "GetAudioLength": (C.c_int, [C.c_char_p]),
    "wavread": (None, [C.c_char_p, _IP, _IP, _P]),
    "WriteF0": (None, [C.c_char_p, C.c_int, C.c_double, _P, _P, C.c_int]),
    "ReadF0": (C.c_int, [C.c_char_p, _P, _P]),
    "GetHeaderInformation": (C.c_double, [C.c_char_p, C.c_char_p]),
    "WriteSpectralEnvelope": (None, [C.c_char_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, _P]),
    "ReadSpectralEnvelope": (C.c_int, [C.c_char_p, _P]),
    "WriteAperiodicity": (None, [C.c_char_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, _P]),
    "ReadAperiodicity": (C.c_int, [C.c_char_p, _P]),
    "world_b200_write_rows": (C.c_int, [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, _P]),
    "world_b200_read_rows": (C.c_int, [C.c_char_p, C.c_char_p, _P, C.c_int]),
    # public MATLAB-style helpers (world/matlabfunctions.h), host only
    "fftshift": (None, [_P, C.c_int, _P]),
    "histc": (None, [_P, C.c_int, _P, C.c_int, _P]),
    "interp1": (None, [_P, _P, C.c_int, _P, C.c_int, _P]),
    "decimate": (None, [_P, C.c_int, C.c_int, _P]),
    "matlab_round": (C.c_int, [C.c_double]),
    "diff": (None, [_P, C.c_int, _P]),
    "interp1Q": (None, [C.c_double, C.c_double, _P, C.c_int, _P, C.c_int, _P]),
    "randn": (C.c_double, [_P]),
    "randn_reseed": (None, [_P]),
    "matlab_std": (C.c_double, [_P, C.c_int]),
    "GetNumberOfAperiodicities": (C.c_int, [C.c_int]),
    "CodeAperiodicity": (None, [_P, C.c_int, C.c_int, C.c_int, _P]),
    "DecodeAperiodicity": (None, [_P, C.c_int, C.c_int, C.c_int, _P]),
    "CodeSpectralEnvelope": (None, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "DecodeSpectralEnvelope": (None, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
}


class WorldError(RuntimeError):
    pass


def load_library(path: str | None = None) -> C.CDLL:
    path = path or os.environ.get("WORLD_B200_LIB") or DEFAULT_LIB
    if not os.path.exists(path):
        raise WorldError(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                         "(nvcc, sm_90a).  There is no CPU fallback.")
    lib = C.CDLL(path)
    for name, (res, args) in ABI.items():
        fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
        fn.restype = res
        fn.argtypes = args
    return lib


def _ptr(a):
    if a is None:
        return None
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    return a.ctypes.data


def _harvest_options(options, n):
    """A list of n HarvestOption (one per utterance) as a ctypes array; None for a single option or None."""
    if options is None or isinstance(options, HarvestOption):
        return None
    options = list(options)
    if len(options) != n:
        raise ValueError(f"{len(options)} Harvest options for {n} utterances")
    arr = (HarvestOption * n)()
    for i, o in enumerate(options):
        arr[i].f0_floor, arr[i].f0_ceil, arr[i].frame_period = o.f0_floor, o.f0_ceil, o.frame_period
    return arr


def _dio_options(options, n):
    """A list of n DioOption (one per utterance) as a ctypes array; None for a single option or None."""
    if options is None or isinstance(options, DioOption):
        return None
    options = list(options)
    if len(options) != n:
        raise ValueError(f"{len(options)} DIO options for {n} utterances")
    arr = (DioOption * n)()
    for i, o in enumerate(options):
        for name, _ in DioOption._fields_:
            setattr(arr[i], name, getattr(o, name))
    return arr


def _chain_options(harvest_options, dio_options, n):
    """The per-utterance options of a chain as (harvest array or None, DIO array or None).  A chain takes the options
    of one F0 method only, as a list of one option per utterance: a single option is refused rather than ignored
    (the chain's own option in the AnalysisOption is the way to give one option for the batch)."""
    if harvest_options is not None and dio_options is not None:
        raise ValueError("harvest_options and dio_options: pass the options of one F0 method")
    if isinstance(harvest_options, HarvestOption) or isinstance(dio_options, DioOption):
        raise TypeError("harvest_options / dio_options: a list of one option per utterance (one option for the batch "
                        "goes into the AnalysisOption)")
    return _harvest_options(harvest_options, n), _dio_options(dio_options, n)


def _pcm16(dtype):
    """True for an int16 dtype (torch.int16, numpy.int16 or "int16"), False for None / float64."""
    name = str(getattr(dtype, "__name__", dtype)).replace("torch.", "")
    if dtype is None or name == "float64":
        return False
    if name == "int16":
        return True
    raise ValueError(f"dtype must be float64 or int16, not {dtype}")


def _int_array(v, n):
    if v is None:
        return None, None
    arr = (C.c_int * n)(*[int(t) for t in v])
    return arr, arr


class World:
    """One analysis context on one GPU.  Method names and argument meaning follow the
    reference's C API; every method takes a batch."""

    def __init__(self, device: int = 0, lib_path: str | None = None, array_module: str = "torch"):
        self.lib = load_library(lib_path)
        self._h = _P()
        rc = self.lib.world_b200_create(device, C.byref(self._h))
        if rc != 0:
            raise WorldError(f"world_b200_create(device={device}) failed with code {rc}: "
                             "a CUDA device is required (no CPU path)")
        self.device = device
        self.xp = array_module
        if array_module == "torch":
            import torch
            self.torch = torch

    # -- plumbing ----------------------------------------------------------------------------
    def close(self):
        if self._h:
            self.lib.world_b200_destroy(self._h)
            self._h = _P()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise WorldError(f"world_b200 error {rc}: {self.lib.world_b200_last_error(self._h).decode()}")

    def _use_current_stream(self):
        if self.xp == "torch":
            s = self.torch.cuda.current_stream(self.device).cuda_stream
            self._check(self.lib.world_b200_set_stream(self._h, _P(s)))

    def _empty(self, like, shape):
        if self.xp == "torch":
            return self.torch.empty(shape, dtype=self.torch.float64, device=like.device)
        import numpy as np
        return np.empty(shape, dtype=np.float64)

    def _zeros(self, like, shape):
        out = self._empty(like, shape)
        if self.xp == "torch":
            out.zero_()
        else:
            out[...] = 0.0
        return out

    def synchronize(self):
        self._check(self.lib.world_b200_synchronize(self._h))

    def trim(self):
        """give back the device memory cached between calls"""
        self._check(self.lib.world_b200_trim(self._h))

    def launch_count(self) -> int:
        return int(self.lib.world_b200_launch_count(self._h))

    def set_scratch_budget(self, nbytes: int):
        self._check(self.lib.world_b200_set_scratch_budget(self._h, nbytes))

    def rfft_test(self, x, out):
        self._use_current_stream()
        self._check(self.lib.world_b200_rfft_test(self._h, _ptr(x), int(x.shape[0]), _ptr(out)))
        return out

    def sfft_test(self, x, out):
        self._use_current_stream()
        self._check(self.lib.world_b200_sfft_test(self._h, _ptr(x), int(x.shape[0]), _ptr(out)))
        return out

    def fp64_peak(self) -> float:
        v = C.c_double(0.0)
        self._check(self.lib.world_b200_fp64_peak(self._h, C.byref(v)))
        return v.value

    def fp64_tensor_peak(self) -> float:
        v = C.c_double(0.0)
        self._check(self.lib.world_b200_fp64_tensor_peak(self._h, C.byref(v)))
        return v.value

    def profile(self, enable=True):
        self._check(self.lib.world_b200_profile(self._h, 1 if enable else 0))

    def profile_report(self) -> dict:
        import json
        buf = C.create_string_buffer(1 << 16)
        self._check(self.lib.world_b200_profile_report(self._h, buf, len(buf)))
        return json.loads(buf.value.decode())

    def randn_stream(self, n_draws, out_u32):
        """test hook: raw draw sums into a uint32 array/tensor of n_draws elements"""
        self._use_current_stream()
        self._check(self.lib.world_b200_randn_stream(self._h, n_draws, _ptr(out_u32)))
        return out_u32

    def randn_window(self, first, n, out_u32):
        """test hook: raw draw sums of draws [first, first + n) into a uint32 array/tensor of n elements"""
        self._use_current_stream()
        self._check(self.lib.world_b200_randn_window(self._h, first, n, _ptr(out_u32)))
        return out_u32

    def frames(self, fs, x_length, frame_period=5.0) -> int:
        return int(self.lib.world_b200_frames(fs, x_length, frame_period))

    # -- options -----------------------------------------------------------------------------
    def dio_option(self) -> DioOption:
        o = DioOption()
        self.lib.InitializeDioOption(C.byref(o))
        return o

    def harvest_option(self) -> HarvestOption:
        o = HarvestOption()
        self.lib.InitializeHarvestOption(C.byref(o))
        return o

    def cheaptrick_option(self, fs) -> CheapTrickOption:
        o = CheapTrickOption()
        self.lib.InitializeCheapTrickOption(fs, C.byref(o))
        return o

    def d4c_option(self) -> D4COption:
        o = D4COption()
        self.lib.InitializeD4COption(C.byref(o))
        return o

    # -- stages ------------------------------------------------------------------------------
    def _f0_stride(self, fs, x, x_lengths, frame_period):
        n, stride = x.shape
        lens = [stride] * n if x_lengths is None else [int(v) for v in x_lengths]
        fl = [self.frames(fs, v, frame_period) for v in lens]
        return max(fl), fl

    def dio(self, x, fs, option=None, x_lengths=None):
        """option: one DioOption for the batch, or a list of one per utterance (f0_floor / f0_ceil /
        channels_in_octave / allowed_range may differ, frame_period and speed may not)."""
        n, stride = x.shape
        per_utt = _dio_options(option, n)
        option = option or self.dio_option()
        frame_period = per_utt[0].frame_period if per_utt is not None and n else getattr(option, "frame_period", 5.0)
        f_stride, fl = self._f0_stride(fs, x, x_lengths, frame_period)
        t = self._zeros(x, (n, f_stride))
        f0 = self._zeros(x, (n, f_stride))
        xl, keep = _int_array(x_lengths, n)
        self._use_current_stream()
        if per_utt is not None:
            self._check(self.lib.world_b200_dio_batch_options(self._h, _ptr(x), n, stride, xl, fs, per_utt,
                                                              _ptr(t), _ptr(f0), f_stride))
        else:
            self._check(self.lib.world_b200_dio_batch(self._h, _ptr(x), n, stride, xl, fs, C.byref(option),
                                                      _ptr(t), _ptr(f0), f_stride))
        return t, f0, fl

    def harvest(self, x, fs, option=None, x_lengths=None):
        """option: one HarvestOption for the batch, or a list of one per utterance (f0_floor / f0_ceil may differ,
        frame_period may not)."""
        n, stride = x.shape
        per_utt = _harvest_options(option, n)
        option = option or self.harvest_option()
        frame_period = per_utt[0].frame_period if per_utt is not None and n else getattr(option, "frame_period", 5.0)
        f_stride, fl = self._f0_stride(fs, x, x_lengths, frame_period)
        t = self._zeros(x, (n, f_stride))
        f0 = self._zeros(x, (n, f_stride))
        xl, keep = _int_array(x_lengths, n)
        self._use_current_stream()
        if per_utt is not None:
            self._check(self.lib.world_b200_harvest_batch_options(self._h, _ptr(x), n, stride, xl, fs, per_utt,
                                                                  _ptr(t), _ptr(f0), f_stride))
        else:
            self._check(self.lib.world_b200_harvest_batch(self._h, _ptr(x), n, stride, xl, fs, C.byref(option),
                                                          _ptr(t), _ptr(f0), f_stride))
        return t, f0, fl

    def stonemask(self, x, fs, time_axis, f0, x_lengths=None, f0_lengths=None):
        n, stride = x.shape
        out = self._zeros(x, tuple(f0.shape))
        xl, k1 = _int_array(x_lengths, n)
        fl, k2 = _int_array(f0_lengths, n)
        self._use_current_stream()
        self._check(self.lib.world_b200_stonemask_batch(self._h, _ptr(x), n, stride, xl, fs, _ptr(time_axis),
                                                        _ptr(f0), fl, f0.shape[1], _ptr(out)))
        return out

    def cheaptrick(self, x, fs, time_axis, f0, option: CheapTrickOption | None = None, x_lengths=None,
                   f0_lengths=None, out=None):
        option = option or self.cheaptrick_option(fs)
        n, stride = x.shape
        bins = option.fft_size // 2 + 1
        if out is None:
            out = self._zeros(x, (n, f0.shape[1], bins))
        xl, k1 = _int_array(x_lengths, n)
        fl, k2 = _int_array(f0_lengths, n)
        self._use_current_stream()
        self._check(self.lib.world_b200_cheaptrick_batch(self._h, _ptr(x), n, stride, xl, fs, _ptr(time_axis),
                                                         _ptr(f0), fl, f0.shape[1], C.byref(option), _ptr(out)))
        return out

    def d4c(self, x, fs, time_axis, f0, fft_size, option: D4COption | None = None, x_lengths=None,
            f0_lengths=None, out=None):
        option = option or self.d4c_option()
        n, stride = x.shape
        bins = fft_size // 2 + 1
        if out is None:
            out = self._zeros(x, (n, f0.shape[1], bins))
        xl, k1 = _int_array(x_lengths, n)
        fl, k2 = _int_array(f0_lengths, n)
        self._use_current_stream()
        self._check(self.lib.world_b200_d4c_batch(self._h, _ptr(x), n, stride, xl, fs, _ptr(time_axis), _ptr(f0),
                                                  fl, f0.shape[1], fft_size, C.byref(option), _ptr(out)))
        return out

    def cheaptrick_coded(self, x, fs, time_axis, f0, number_of_dimensions, option: CheapTrickOption | None = None,
                         x_lengths=None, f0_lengths=None):
        """CheapTrick + CodeSpectralEnvelope in one kernel per frame -> [n, L, number_of_dimensions]."""
        option = option or self.cheaptrick_option(fs)
        n, stride = x.shape
        out = self._zeros(x, (n, f0.shape[1], number_of_dimensions))
        xl, k1 = _int_array(x_lengths, n)
        fl, k2 = _int_array(f0_lengths, n)
        self._use_current_stream()
        self._check(self.lib.world_b200_cheaptrick_coded_batch(self._h, _ptr(x), n, stride, xl, fs, _ptr(time_axis),
                                                               _ptr(f0), fl, f0.shape[1], C.byref(option),
                                                               number_of_dimensions, _ptr(out)))
        return out

    def d4c_coded(self, x, fs, time_axis, f0, fft_size, option: D4COption | None = None, x_lengths=None,
                  f0_lengths=None):
        """D4C + CodeAperiodicity in one kernel per frame -> [n, L, GetNumberOfAperiodicities(fs)]."""
        option = option or self.d4c_option()
        n, stride = x.shape
        out = self._zeros(x, (n, f0.shape[1], max(1, self.number_of_aperiodicities(fs))))
        xl, k1 = _int_array(x_lengths, n)
        fl, k2 = _int_array(f0_lengths, n)
        self._use_current_stream()
        self._check(self.lib.world_b200_d4c_coded_batch(self._h, _ptr(x), n, stride, xl, fs, _ptr(time_axis), _ptr(f0),
                                                        fl, f0.shape[1], fft_size, C.byref(option), _ptr(out)))
        return out

    def synthesis(self, f0, spectrogram, aperiodicity, fft_size, frame_period, fs, y_length, f0_lengths=None,
                  y_lengths=None):
        """Batched Synthesis(): f0 [n, L], spectrogram / aperiodicity [n, L, bins] -> y [n, y_length]."""
        n = f0.shape[0]
        y = self._zeros(f0, (n, y_length))
        fl, k1 = _int_array(f0_lengths, n)
        yl, k2 = _int_array(y_lengths, n)
        self._use_current_stream()
        self._check(self.lib.world_b200_synthesis_batch(self._h, _ptr(f0), fl, n, f0.shape[1], _ptr(spectrogram),
                                                        _ptr(aperiodicity), fft_size, frame_period, fs, yl, y_length,
                                                        _ptr(y)))
        return y

    def synthesis_coded(self, f0, coded_spectral_envelope, coded_aperiodicity, fft_size, frame_period, fs, y_length,
                        f0_lengths=None, y_lengths=None, dtype=None):
        """Batched Synthesis() from coded rows: f0 [n, L], coded_spectral_envelope [n, L, number_of_dimensions],
        coded_aperiodicity [n, L, GetNumberOfAperiodicities(fs)] -> y [n, y_length].  The rows are decoded chunk by
        chunk inside the call; the output equals decode_spectral_envelope + decode_aperiodicity + synthesis bit for
        bit.  coded_aperiodicity may be None below 12 kHz (no bands).  dtype: float64 (default) for the waveform, or
        int16 for its 16-bit PCM, quantised as wavwrite does by the overlap-add kernel itself."""
        pcm16 = _pcm16(dtype)
        n = f0.shape[0]
        if pcm16 and self.xp == "torch":
            y = self.torch.zeros((n, y_length), dtype=self.torch.int16, device=f0.device)
        elif pcm16:
            import numpy as np
            y = np.zeros((n, y_length), dtype=np.int16)
        else:
            y = self._zeros(f0, (n, y_length))
        fl, k1 = _int_array(f0_lengths, n)
        yl, k2 = _int_array(y_lengths, n)
        fn = self.lib.world_b200_synthesis_coded_batch_pcm16 if pcm16 else self.lib.world_b200_synthesis_coded_batch
        self._use_current_stream()
        self._check(fn(self._h, _ptr(f0), fl, n, f0.shape[1], _ptr(coded_spectral_envelope),
                       int(coded_spectral_envelope.shape[-1]), _ptr(coded_aperiodicity), fft_size, frame_period, fs,
                       yl, y_length, _ptr(y)))
        return y

    def synthesis_coded_host(self, f0, coded_sp, coded_ap, fft_size, frame_period, fs, y_length, nbit=16,
                             f0_lengths=None, y_lengths=None, out=None):
        """synthesis_coded for HOST arrays (numpy arrays or CPU tensors, float64): upload, synthesis and download are
        pipelined over utterance chunks (world_b200_synthesis_coded_host).  Returns y [n, y_length] as a numpy array,
        int16 for nbit 16 or float64 for nbit 0, whole rows (samples beyond an utterance's y_length are 0).  out: a
        host array of that shape and dtype to write into (a pinned one lets the downloads overlap the kernels).
        coded_ap may be None below 12 kHz (no bands)."""
        import numpy as np

        def host(a):
            if a is None:
                return None
            if hasattr(a, "numpy"):
                a = a.detach().numpy()
            return np.ascontiguousarray(a, dtype=np.float64)

        f0, coded_sp, coded_ap = host(f0), host(coded_sp), host(coded_ap)
        n = f0.shape[0]
        if out is None:
            out = np.empty((n, y_length), dtype=np.int16 if nbit == 16 else np.float64)
        y = out.numpy() if hasattr(out, "numpy") else out
        if nbit in (0, 16) and (y.shape != (n, y_length) or y.dtype != (np.int16 if nbit == 16 else np.float64)
                                or not y.flags.c_contiguous):
            raise ValueError(f"out: a contiguous [{n}, {y_length}] {'int16' if nbit == 16 else 'float64'} host array")
        fl, k1 = _int_array(f0_lengths, n)
        yl, k2 = _int_array(y_lengths, n)
        self._check(self.lib.world_b200_synthesis_coded_host(self._h, _ptr(f0), fl, n, f0.shape[1], _ptr(coded_sp),
                                                             int(coded_sp.shape[-1]), _ptr(coded_ap), fft_size,
                                                             frame_period, fs, yl, y_length, nbit, _ptr(y)))
        return y

    def analysis_option(self, fs, f0_method=F0_HARVEST) -> AnalysisOption:
        o = AnalysisOption()
        self.lib.world_b200_default_analysis_option(fs, f0_method, C.byref(o))
        return o

    def analyze_batch(self, x, fs, option: AnalysisOption, x_lengths=None, time_axis=None, f0=None,
                      spectrogram=None, aperiodicity=None, harvest_options=None, dio_options=None):
        """Whole chain on DEVICE arrays in one call (two internal streams); returns (t, f0, sp, ap, frame counts).
        harvest_options: a list of one HarvestOption per utterance (Harvest with a per-utterance F0 range);
        dio_options: a list of one DioOption per utterance (DIO + StoneMask with a per-utterance F0 range)."""
        n, stride = x.shape
        frame_period = option.dio.frame_period if option.f0_method == F0_DIO_STONEMASK else option.harvest.frame_period
        f_stride, fl = self._f0_stride(fs, x, x_lengths, frame_period)
        bins = option.cheaptrick.fft_size // 2 + 1
        if time_axis is None:
            time_axis = self._zeros(x, (n, f_stride))
        if f0 is None:
            f0 = self._zeros(x, (n, f_stride))
        if spectrogram is None:
            spectrogram = self._zeros(x, (n, f_stride, bins))
        if aperiodicity is None:
            aperiodicity = self._zeros(x, (n, f_stride, bins))
        xl, keep = _int_array(x_lengths, n)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        self._use_current_stream()
        if per_utt is not None:
            self._check(self.lib.world_b200_analyze_batch_options(self._h, _ptr(x), n, stride, xl, fs, C.byref(option),
                                                                  per_utt, _ptr(time_axis), _ptr(f0),
                                                                  time_axis.shape[1], _ptr(spectrogram),
                                                                  _ptr(aperiodicity)))
        elif per_dio is not None:
            self._check(self.lib.world_b200_analyze_batch_dio_options(self._h, _ptr(x), n, stride, xl, fs,
                                                                      C.byref(option), per_dio, _ptr(time_axis),
                                                                      _ptr(f0), time_axis.shape[1], _ptr(spectrogram),
                                                                      _ptr(aperiodicity)))
        else:
            self._check(self.lib.world_b200_analyze_batch(self._h, _ptr(x), n, stride, xl, fs, C.byref(option),
                                                          _ptr(time_axis), _ptr(f0), time_axis.shape[1],
                                                          _ptr(spectrogram), _ptr(aperiodicity)))
        return time_axis, f0, spectrogram, aperiodicity, fl

    # -- multi-GPU: one World per GPU / process; the NCCL id travels by the caller's own means -------------------
    def comm_unique_id(self) -> bytes:
        buf = (C.c_ubyte * 128)()
        rc = self.lib.world_b200_comm_unique_id(buf, 128)
        if rc:
            raise WorldError(f"world_b200_comm_unique_id failed ({rc}): NCCL not available")
        return bytes(buf)

    def comm_init(self, n_ranks: int, rank: int, unique_id: bytes):
        buf = (C.c_ubyte * 128).from_buffer_copy(unique_id[:128])
        self._check(self.lib.world_b200_comm_init(self._h, n_ranks, rank, buf, 128))

    def comm_destroy(self):
        self._check(self.lib.world_b200_comm_destroy(self._h))

    def allgather_rows(self, full, rows_per_rank: int):
        """In-place all-gather of [n_ranks * rows_per_rank, ...] (this rank's block already written)."""
        row_elems = 1
        for d in full.shape[1:]:
            row_elems *= int(d)
        self._use_current_stream()
        self._check(self.lib.world_b200_allgather_rows(self._h, _ptr(full), row_elems, rows_per_rank))
        return full

    def analyze_batch_allgather(self, x, fs, option: AnalysisOption, time_axis_full, f0_full, spectrogram_full,
                                aperiodicity_full, x_lengths=None, harvest_options=None, dio_options=None):
        """analyze_batch on this rank's shard with every finished slice broadcast into the FULL arrays of all ranks.
        harvest_options / dio_options: a list of one option per utterance of THIS rank's shard."""
        n, stride = x.shape
        xl, keep = _int_array(x_lengths, n)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        outs = (_ptr(time_axis_full), _ptr(f0_full), time_axis_full.shape[1],
                _ptr(spectrogram_full) if spectrogram_full is not None else None,
                _ptr(aperiodicity_full) if aperiodicity_full is not None else None)
        self._use_current_stream()
        if per_utt is not None:
            self._check(self.lib.world_b200_analyze_batch_allgather_options(
                self._h, _ptr(x), n, stride, xl, fs, C.byref(option), per_utt, *outs))
        elif per_dio is not None:
            self._check(self.lib.world_b200_analyze_batch_allgather_dio_options(
                self._h, _ptr(x), n, stride, xl, fs, C.byref(option), per_dio, *outs))
        else:
            self._check(self.lib.world_b200_analyze_batch_allgather(
                self._h, _ptr(x), n, stride, xl, fs, C.byref(option), *outs))

    def analyze_host(self, x_host, fs, option: AnalysisOption, x_lengths=None, time_axis=None, f0=None,
                     spectrogram=None, aperiodicity=None, f0_stride=None, harvest_options=None, dio_options=None):
        """Whole chain on HOST arrays (numpy or pinned torch CPU tensors); outputs are written
        into the given host arrays (allocated with numpy when None).  harvest_options / dio_options: a list of
        one option per utterance of the chain's F0 method."""
        import numpy as np
        n, stride = x_host.shape
        frame_period = option.dio.frame_period if option.f0_method == F0_DIO_STONEMASK else option.harvest.frame_period
        lens = [stride] * n if x_lengths is None else [int(v) for v in x_lengths]
        fl = [self.frames(fs, v, frame_period) for v in lens]
        f0_stride = f0_stride or max(fl)
        bins = option.cheaptrick.fft_size // 2 + 1
        if time_axis is None:
            time_axis = np.zeros((n, f0_stride))
        if f0 is None:
            f0 = np.zeros((n, f0_stride))
        if spectrogram is None:
            spectrogram = np.zeros((n, f0_stride, bins))
        if aperiodicity is None:
            aperiodicity = np.zeros((n, f0_stride, bins))
        xl, keep = _int_array(x_lengths, n)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        if per_utt is not None:
            self._check(self.lib.world_b200_analyze_host_options(self._h, _ptr(x_host), n, stride, xl, fs,
                                                                 C.byref(option), per_utt, _ptr(time_axis), _ptr(f0),
                                                                 f0_stride, _ptr(spectrogram), _ptr(aperiodicity)))
        elif per_dio is not None:
            self._check(self.lib.world_b200_analyze_host_dio_options(self._h, _ptr(x_host), n, stride, xl, fs,
                                                                     C.byref(option), per_dio, _ptr(time_axis),
                                                                     _ptr(f0), f0_stride, _ptr(spectrogram),
                                                                     _ptr(aperiodicity)))
        else:
            self._check(self.lib.world_b200_analyze_host(self._h, _ptr(x_host), n, stride, xl, fs, C.byref(option),
                                                         _ptr(time_axis), _ptr(f0), f0_stride, _ptr(spectrogram),
                                                         _ptr(aperiodicity)))
        return time_axis, f0, spectrogram, aperiodicity, fl

    # -- codec (codec.h) and ingest ----------------------------------------------------------
    def number_of_aperiodicities(self, fs) -> int:
        return int(self.lib.GetNumberOfAperiodicities(fs))

    def _codec(self, fn, src, out_width, fs, fft_size, f0_lengths, dims=None):
        n, stride = src.shape[0], src.shape[1]
        out = self._zeros(src, (n, stride, out_width))
        fl, keep = _int_array(f0_lengths, n)
        self._use_current_stream()
        args = [self._h, _ptr(src), n, fl, stride, fs, fft_size]
        if dims is not None:
            args.append(dims)
        self._check(fn(*args, _ptr(out)))
        return out

    def code_aperiodicity(self, aperiodicity, fs, fft_size, f0_lengths=None):
        return self._codec(self.lib.world_b200_code_aperiodicity_batch, aperiodicity,
                           max(1, self.number_of_aperiodicities(fs)), fs, fft_size, f0_lengths)

    def decode_aperiodicity(self, coded, fs, fft_size, f0_lengths=None):
        return self._codec(self.lib.world_b200_decode_aperiodicity_batch, coded, fft_size // 2 + 1, fs, fft_size,
                           f0_lengths)

    def code_spectral_envelope(self, spectrogram, fs, fft_size, number_of_dimensions, f0_lengths=None):
        return self._codec(self.lib.world_b200_code_spectral_envelope_batch, spectrogram, number_of_dimensions, fs,
                           fft_size, f0_lengths, number_of_dimensions)

    def decode_spectral_envelope(self, coded, fs, fft_size, number_of_dimensions, f0_lengths=None):
        return self._codec(self.lib.world_b200_decode_spectral_envelope_batch, coded, fft_size // 2 + 1, fs,
                           fft_size, f0_lengths, number_of_dimensions)

    def wav_parse(self, data: bytes):
        """Host only: (fs, nbit, n_samples, data_offset) of a mono PCM WAV image."""
        fs, nbit, ns, off = C.c_int(), C.c_int(), C.c_int(), C.c_ulonglong()
        buf = (C.c_ubyte * len(data)).from_buffer_copy(data)
        rc = self.lib.world_b200_wav_parse(buf, len(data), C.byref(fs), C.byref(nbit), C.byref(ns), C.byref(off))
        if rc != 0:
            raise WorldError(f"not a mono PCM WAV image the reference's wavread accepts (code {rc})")
        return fs.value, nbit.value, ns.value, off.value

    def pcm_to_double(self, pcm, nbit, x_lengths=None):
        """pcm: [n, stride * nbit/8] uint8 (or [n, stride] int16 for nbit 16) on the device -> doubles."""
        n = pcm.shape[0]
        stride = pcm.shape[1] * pcm.element_size() // (nbit // 8) if hasattr(pcm, "element_size") \
            else pcm.shape[1] * pcm.itemsize // (nbit // 8)
        if self.xp == "torch":
            x = self.torch.zeros((n, stride), dtype=self.torch.float64, device=pcm.device)
        else:
            import numpy as np
            x = np.zeros((n, stride))
        xl, keep = _int_array(x_lengths, n)
        self._use_current_stream()
        self._check(self.lib.world_b200_pcm_to_double_batch(self._h, _ptr(pcm), nbit, n, stride, xl, _ptr(x)))
        return x

    def analyze_coded_host(self, x_host, nbit, fs, option: AnalysisOption, number_of_dimensions, x_lengths=None,
                           time_axis=None, f0=None, coded_sp=None, coded_ap=None, f0_stride=None, harvest_options=None,
                           dio_options=None):
        """Whole chain with device-side ingest (nbit 0 = float64 rows, 16 = int16 rows, ...) and codec;
        only the coded rows are downloaded.  harvest_options / dio_options: a list of one option per utterance of
        the chain's F0 method (not both)."""
        import numpy as np
        n = x_host.shape[0]
        item = x_host.element_size() if hasattr(x_host, "element_size") else x_host.itemsize
        stride = x_host.shape[1] * item // (nbit // 8 if nbit else 8)
        frame_period = option.dio.frame_period if option.f0_method == F0_DIO_STONEMASK else option.harvest.frame_period
        lens = [stride] * n if x_lengths is None else [int(v) for v in x_lengths]
        fl = [self.frames(fs, v, frame_period) for v in lens]
        f0_stride = f0_stride or max(fl)
        n_ap = self.number_of_aperiodicities(fs)
        if time_axis is None:
            time_axis = np.zeros((n, f0_stride))
        if f0 is None:
            f0 = np.zeros((n, f0_stride))
        if coded_sp is None:
            coded_sp = np.zeros((n, f0_stride, number_of_dimensions))
        if coded_ap is None:
            coded_ap = np.zeros((n, f0_stride, max(1, n_ap)))
        xl, keep = _int_array(x_lengths, n)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        outs = (number_of_dimensions, _ptr(time_axis), _ptr(f0), f0_stride, _ptr(coded_sp), _ptr(coded_ap))
        if per_utt is not None:
            self._check(self.lib.world_b200_analyze_coded_host_options(self._h, _ptr(x_host), nbit, n, stride, xl, fs,
                                                                       C.byref(option), per_utt, *outs))
        elif per_dio is not None:
            self._check(self.lib.world_b200_analyze_coded_host_dio_options(self._h, _ptr(x_host), nbit, n, stride, xl,
                                                                           fs, C.byref(option), per_dio, *outs))
        else:
            self._check(self.lib.world_b200_analyze_coded_host(self._h, _ptr(x_host), nbit, n, stride, xl, fs,
                                                               C.byref(option), *outs))
        return time_axis, f0, coded_sp, coded_ap, fl

    def _coded_rows(self, x, nbit, option):
        """(n, row stride in samples, frame_period) of a coded chain's input: float64 rows for nbit 0, else PCM rows
        of nbit/8 bytes per sample held in any integer dtype (int16 for 16-bit, uint8 rows for 8/24/32-bit)."""
        if nbit not in (0, 8, 16, 24, 32):
            raise ValueError(f"nbit must be 0, 8, 16, 24 or 32, not {nbit}")
        item = x.element_size() if hasattr(x, "element_size") else x.itemsize
        width = nbit // 8 if nbit else 8
        if (x.shape[1] * item) % width:
            raise ValueError(f"rows of {x.shape[1] * item} bytes do not hold whole {width}-byte samples")
        frame_period = option.dio.frame_period if option.f0_method == F0_DIO_STONEMASK else option.harvest.frame_period
        return x.shape[0], x.shape[1] * item // width, frame_period

    def analyze_coded_batch(self, x, nbit, fs, option: AnalysisOption, number_of_dimensions, x_lengths=None,
                            time_axis=None, f0=None, coded_sp=None, coded_ap=None, harvest_options=None,
                            dio_options=None):
        """Whole chain on DEVICE arrays with coded rows out: analyze_batch's two internal streams, analyze_coded_host's
        formats.  x: float64 rows (nbit 0) or PCM rows (nbit 16: int16; 8/24/32: uint8 rows of nbit/8 bytes per
        sample); the PCM is converted slice by slice on the device.  Outputs are allocated on x's device when None
        and the work is enqueued on torch's current stream.  Returns (t, f0, coded_sp, coded_ap, frame counts) with
        coded_sp [n, L, number_of_dimensions] and coded_ap [n, L, max(1, GetNumberOfAperiodicities(fs))] (left zero
        below 12 kHz).  harvest_options / dio_options: a list of one option per utterance of the chain's F0 method."""
        n, stride, frame_period = self._coded_rows(x, nbit, option)
        lens = [stride] * n if x_lengths is None else [int(v) for v in x_lengths]
        fl = [self.frames(fs, v, frame_period) for v in lens]
        f_stride = max(fl) if fl else 1
        if time_axis is None:
            time_axis = self._zeros(x, (n, f_stride))
        if f0 is None:
            f0 = self._zeros(x, (n, f_stride))
        if coded_sp is None:
            coded_sp = self._zeros(x, (n, f_stride, number_of_dimensions))
        if coded_ap is None:
            coded_ap = self._zeros(x, (n, f_stride, max(1, self.number_of_aperiodicities(fs))))
        xl, keep = _int_array(x_lengths, n)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        outs = (number_of_dimensions, _ptr(time_axis), _ptr(f0), time_axis.shape[1], _ptr(coded_sp), _ptr(coded_ap))
        self._use_current_stream()
        if per_utt is not None:
            self._check(self.lib.world_b200_analyze_coded_batch_options(self._h, _ptr(x), nbit, n, stride, xl, fs,
                                                                        C.byref(option), per_utt, *outs))
        elif per_dio is not None:
            self._check(self.lib.world_b200_analyze_coded_batch_dio_options(self._h, _ptr(x), nbit, n, stride, xl, fs,
                                                                            C.byref(option), per_dio, *outs))
        else:
            self._check(self.lib.world_b200_analyze_coded_batch(self._h, _ptr(x), nbit, n, stride, xl, fs,
                                                                C.byref(option), *outs))
        return time_axis, f0, coded_sp, coded_ap, fl

    def analyze_coded_batch_allgather(self, x, nbit, fs, option: AnalysisOption, number_of_dimensions, time_axis_full,
                                      f0_full, coded_sp_full, coded_ap_full, x_lengths=None, harvest_options=None,
                                      dio_options=None):
        """analyze_coded_batch on this rank's shard with every finished slice sent into the FULL arrays of all ranks
        (the coded rows are what crosses between GPUs).  coded_sp_full / coded_ap_full may be None to skip CheapTrick /
        D4C.  harvest_options / dio_options: a list of one option per utterance of THIS rank's shard."""
        n, stride, _ = self._coded_rows(x, nbit, option)
        xl, keep = _int_array(x_lengths, n)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        outs = (number_of_dimensions, _ptr(time_axis_full), _ptr(f0_full), time_axis_full.shape[1],
                _ptr(coded_sp_full), _ptr(coded_ap_full))
        self._use_current_stream()
        if per_utt is not None:
            self._check(self.lib.world_b200_analyze_coded_batch_allgather_options(
                self._h, _ptr(x), nbit, n, stride, xl, fs, C.byref(option), per_utt, *outs))
        elif per_dio is not None:
            self._check(self.lib.world_b200_analyze_coded_batch_allgather_dio_options(
                self._h, _ptr(x), nbit, n, stride, xl, fs, C.byref(option), per_dio, *outs))
        else:
            self._check(self.lib.world_b200_analyze_coded_batch_allgather(
                self._h, _ptr(x), nbit, n, stride, xl, fs, C.byref(option), *outs))
