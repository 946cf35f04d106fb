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
_LP = C.POINTER(C.c_longlong)

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
    "world_b200_cheaptrick_batch_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP, C.c_int,
                                                      C.POINTER(CheapTrickOption), C.c_int, _P]),
    "world_b200_d4c_batch_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP, C.c_int, _IP,
                                               C.POINTER(D4COption), C.c_int, _P]),
    "world_b200_cheaptrick_coded_batch_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP,
                                                            C.c_int, C.POINTER(CheapTrickOption), C.c_int, _P]),
    "world_b200_d4c_coded_batch_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int, _P, _P, _IP, C.c_int,
                                                     _IP, C.POINTER(D4COption), _P]),
    "world_b200_synthesis_batch": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, _P, C.c_int, C.c_double, C.c_int, _IP,
                                             C.c_int, _P]),
    "world_b200_synthesis_coded_batch": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_double,
                                                   C.c_int, _IP, C.c_int, _P]),
    "world_b200_synthesis_coded_batch_pcm16": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int,
                                                         C.c_double, C.c_int, _IP, C.c_int, _P]),
    "world_b200_synthesis_coded_host": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_double,
                                                  C.c_int, _IP, C.c_int, C.c_int, _P]),
    "world_b200_modify_batch": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P]),
    "world_b200_synthesis_coded_batch_modified": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int,
                                                            C.c_double, C.c_int, _IP, C.c_int, _P, _P, C.c_int, _P]),
    "world_b200_synthesis_coded_host_modified": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int,
                                                           C.c_double, C.c_int, _IP, C.c_int, _P, _P, C.c_int, _P]),
    "world_b200_synthesis_batch_options": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, _P, C.c_int, _IP, C.c_double,
                                                     C.c_int, _IP, C.c_int, _P]),
    "world_b200_synthesis_coded_batch_options": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, _IP,
                                                           C.c_double, C.c_int, _IP, C.c_int, _P, _P, C.c_int, _P]),
    "world_b200_synthesis_coded_host_options": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _P, _IP,
                                                          C.c_double, C.c_int, _IP, C.c_int, _P, _P, C.c_int, _P]),
    "world_b200_modify_batch_options": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _IP, C.c_int, _P, _P]),
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
    "world_b200_analyze_batch_spectral_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int,
                                                            C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                            C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                            C.POINTER(D4COption), _P, _P, C.c_int, C.c_int, _P, _P]),
    "world_b200_analyze_host_spectral_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int,
                                                           C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                           C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                           C.POINTER(D4COption), _P, _P, C.c_int, C.c_int, _P, _P]),
    "world_b200_analyze_batch_allgather_spectral_options": (C.c_int, [_P, _P, C.c_int, C.c_int, _IP, C.c_int,
                                                                      C.POINTER(AnalysisOption),
                                                                      C.POINTER(HarvestOption), C.POINTER(DioOption),
                                                                      C.POINTER(CheapTrickOption),
                                                                      C.POINTER(D4COption), _P, _P, C.c_int, C.c_int,
                                                                      _P, _P]),
    # packed batches: x_offsets / f_offsets are n + 1 64-bit offsets
    "world_b200_packed_frames": (C.c_int, [C.c_int, C.c_int, _LP, C.c_double, _LP]),
    "world_b200_analyze_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, C.POINTER(AnalysisOption),
                                            C.POINTER(HarvestOption), C.POINTER(DioOption),
                                            C.POINTER(CheapTrickOption), C.POINTER(D4COption), _P, _P, C.c_int, _P,
                                            _P, _LP]),
    "world_b200_analyze_host_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, C.POINTER(AnalysisOption),
                                                 C.POINTER(HarvestOption), C.POINTER(DioOption),
                                                 C.POINTER(CheapTrickOption), C.POINTER(D4COption), _P, _P, C.c_int,
                                                 _P, _P, _LP]),
    "world_b200_analyze_coded_packed": (C.c_int, [_P, _P, C.c_int, C.c_int, _LP, C.c_int, C.POINTER(AnalysisOption),
                                                  C.POINTER(HarvestOption), C.POINTER(DioOption),
                                                  C.POINTER(CheapTrickOption), C.POINTER(D4COption), C.c_int, _P, _P,
                                                  _P, _P, _LP]),
    "world_b200_analyze_coded_host_packed": (C.c_int, [_P, _P, C.c_int, C.c_int, _LP, C.c_int,
                                                       C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                       C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                       C.POINTER(D4COption), C.c_int, _P, _P, _P, _P, _LP]),
    "world_b200_synthesis_packed": (C.c_int, [_P, _P, C.c_int, _LP, _P, _P, C.c_int, _IP, C.c_double, C.c_int, _LP,
                                              _P]),
    "world_b200_synthesis_coded_packed": (C.c_int, [_P, _P, C.c_int, _LP, _P, C.c_int, _P, _IP, C.c_double, C.c_int,
                                                    _LP, _P, _P, C.c_int, _P]),
    "world_b200_synthesis_coded_host_packed": (C.c_int, [_P, _P, C.c_int, _LP, _P, C.c_int, _P, _IP, C.c_double,
                                                         C.c_int, _LP, _P, _P, C.c_int, _P]),
    "world_b200_modify_packed": (C.c_int, [_P, _P, C.c_int, _LP, _P, C.c_int, _IP, C.c_int, _P, _P]),
    "world_b200_modify_curves": (C.c_int, [_P, _P, _IP, C.c_int, C.c_int, _P, C.c_int, _IP, C.c_int, _P, _P]),
    "world_b200_modify_curves_packed": (C.c_int, [_P, _P, C.c_int, _LP, _P, C.c_int, _IP, C.c_int, _P, _P]),
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
    "world_b200_analyze_coded_host_spectral_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                                 C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                                 C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                                 C.POINTER(D4COption), C.c_int, _P, _P, C.c_int, _P,
                                                                 _P]),
    "world_b200_analyze_coded_batch_spectral_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                                  C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                                  C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                                  C.POINTER(D4COption), C.c_int, _P, _P, C.c_int, _P,
                                                                  _P]),
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
    "world_b200_analyze_coded_batch_allgather_spectral_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP,
                                                                            C.c_int, C.POINTER(AnalysisOption),
                                                                            C.POINTER(HarvestOption),
                                                                            C.POINTER(DioOption),
                                                                            C.POINTER(CheapTrickOption),
                                                                            C.POINTER(D4COption), C.c_int, _P, _P,
                                                                            C.c_int, _P, _P]),
    "world_b200_transform_samples": (C.c_int, [C.c_int, C.c_int, C.c_double, C.c_double]),
    "world_b200_transform_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(AnalysisOption),
                                             C.POINTER(HarvestOption), C.POINTER(DioOption), _P, _P, _P, C.c_int, _P,
                                             C.c_int, _IP]),
    "world_b200_transform_host": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int, C.POINTER(AnalysisOption),
                                            C.POINTER(HarvestOption), C.POINTER(DioOption), _P, _P, _P, C.c_int, _P,
                                            C.c_int, _IP]),
    "world_b200_transform_batch_spectral_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                              C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                              C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                              C.POINTER(D4COption), _P, _P, _P, C.c_int, _P, C.c_int,
                                                              _IP]),
    "world_b200_transform_host_spectral_options": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _IP, C.c_int,
                                                             C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                             C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                             C.POINTER(D4COption), _P, _P, _P, C.c_int, _P, C.c_int,
                                                             _IP]),
    "world_b200_transform_packed_samples": (C.c_int, [C.c_int, C.c_int, _LP, C.c_double, _P, _LP]),
    "world_b200_transform_packed": (C.c_int, [_P, _P, C.c_int, C.c_int, _LP, C.c_int, C.POINTER(AnalysisOption),
                                              C.POINTER(HarvestOption), C.POINTER(DioOption),
                                              C.POINTER(CheapTrickOption), C.POINTER(D4COption), _P, _P, _P, C.c_int,
                                              _P, _LP]),
    "world_b200_transform_host_packed": (C.c_int, [_P, _P, C.c_int, C.c_int, _LP, C.c_int, C.POINTER(AnalysisOption),
                                                   C.POINTER(HarvestOption), C.POINTER(DioOption),
                                                   C.POINTER(CheapTrickOption), C.POINTER(D4COption), _P, _P, _P,
                                                   C.c_int, _P, _LP]),
    "world_b200_transform_packed_curves": (C.c_int, [_P, _P, C.c_int, C.c_int, _LP, C.c_int,
                                                     C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                     C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                     C.POINTER(D4COption), _P, _P, _P, C.c_int, _P, _LP]),
    "world_b200_transform_host_packed_curves": (C.c_int, [_P, _P, C.c_int, C.c_int, _LP, C.c_int,
                                                          C.POINTER(AnalysisOption), C.POINTER(HarvestOption),
                                                          C.POINTER(DioOption), C.POINTER(CheapTrickOption),
                                                          C.POINTER(D4COption), _P, _P, _P, C.c_int, _P, _LP]),
    "world_b200_stonemask_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _P, _P, _LP, _P]),
    "world_b200_cheaptrick_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _P, _P, _LP, C.POINTER(CheapTrickOption),
                                               C.c_int, _P]),
    "world_b200_cheaptrick_coded_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _P, _P, _LP,
                                                     C.POINTER(CheapTrickOption), C.c_int, _P]),
    "world_b200_d4c_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _P, _P, _LP, _IP, C.POINTER(D4COption), C.c_int,
                                        _P]),
    "world_b200_d4c_coded_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _P, _P, _LP, _IP, C.POINTER(D4COption),
                                              _P]),
    "world_b200_code_spectral_envelope_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _IP, C.c_int, C.c_int, _P]),
    "world_b200_decode_spectral_envelope_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _IP, C.c_int, C.c_int, _P]),
    "world_b200_code_aperiodicity_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _IP, C.c_int, _P]),
    "world_b200_decode_aperiodicity_packed": (C.c_int, [_P, _P, C.c_int, _LP, C.c_int, _IP, C.c_int, _P]),
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


def _option_array(cls, options, n):
    """A list of n options of ctypes type cls (one per utterance) as a ctypes array."""
    options = list(options)
    if len(options) != n:
        raise ValueError(f"{len(options)} {cls.__name__} entries for {n} utterances")
    arr = (cls * n)()
    for i, o in enumerate(options):
        C.memmove(C.byref(arr[i]), C.byref(o), C.sizeof(cls))
    return arr


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


def _full_bins(option, cheaptrick_options):
    """Values per frame of the full rows a chain allocates: the largest fft_size // 2 + 1 of cheaptrick_options, or
    option's with one CheapTrick option."""
    sizes = [o.fft_size for o in cheaptrick_options or []] or [option.cheaptrick.fft_size]
    return max(sizes) // 2 + 1


def _row_stride(spectrogram, aperiodicity):
    """The row_stride of a full-row chain with per-utterance spectral options: the last dimension of its spectrogram
    and aperiodicity arrays (the same for both; one may be None, not both)."""
    widths = {int(a.shape[-1]) for a in (spectrogram, aperiodicity) if a is not None}
    if not widths:
        raise ValueError("per-utterance spectral options need the spectrogram or aperiodicity array: its last "
                         "dimension is the row_stride")
    if len(widths) > 1:
        raise ValueError(f"spectrogram and aperiodicity share one row_stride, not {sorted(widths)}")
    return widths.pop()


def _frame_period(option):
    """The frame period of an AnalysisOption's F0 method."""
    return option.dio.frame_period if option.f0_method == F0_DIO_STONEMASK else option.harvest.frame_period


def _pcm16(dtype):
    """True for an int16 dtype (torch.int16, numpy.int16 or "int16"), False for None / float64."""
    name = str(getattr(dtype, "__name__", dtype)).replace("torch.", "")
    if dtype is None or name == "float64":
        return False
    if name == "int16":
        return True
    raise ValueError(f"dtype must be float64 or int16, not {dtype}")


def _factors(v, n, what):
    """None, one factor for every utterance, or a sequence of n factors -> a ctypes double array (or None)."""
    if v is None:
        return None
    if hasattr(v, "tolist"):
        v = v.tolist()
    if isinstance(v, (int, float)):
        v = [v] * n
    v = [float(t) for t in v]
    if len(v) != n:
        raise ValueError(f"{what}: {len(v)} factors for {n} utterances")
    return (C.c_double * n)(*v)


def _offsets(x_offsets):
    """n + 1 sample offsets (a list, numpy array or CPU tensor) -> (n, ctypes int64 array)."""
    if hasattr(x_offsets, "tolist"):
        x_offsets = x_offsets.tolist()
    v = [int(t) for t in x_offsets]
    if not v:
        raise ValueError("x_offsets needs n_utts + 1 entries")
    return len(v) - 1, (C.c_longlong * len(v))(*v)


def _int_array(v, n):
    if v is None:
        return None, None
    arr = (C.c_int * n)(*[int(t) for t in v])
    return arr, arr


def _fft_sizes(fft_size, n):
    """A sequence of n sizes (one per utterance) as a ctypes int array; None for a single size."""
    if not isinstance(fft_size, (list, tuple)) and getattr(fft_size, "ndim", 0) == 0:
        return None
    sizes = fft_size.tolist() if hasattr(fft_size, "tolist") else list(fft_size)
    if len(sizes) != n:
        raise ValueError(f"{len(sizes)} fft sizes for {n} utterances")
    return (C.c_int * max(n, 1))(*[int(v) for v in sizes])


def _curve_sizes(fft_size, n):
    """One size, or a sequence of n sizes -> a ctypes int array of one size per utterance."""
    sizes = _fft_sizes(fft_size, n)
    return (C.c_int * max(n, 1))(*([int(fft_size)] * n)) if sizes is None else sizes


def _curve(c):
    """A curve of float64 factors in its array's memory (tensor or numpy array, contiguous) -> its address, or None."""
    if c is None:
        return None
    tensor = hasattr(c, "data_ptr")
    if str(c.dtype) not in ("float64", "torch.float64") or not (c.is_contiguous() if tensor else c.flags.c_contiguous):
        raise ValueError("a curve: a contiguous float64 array")
    return c.data_ptr() if tensor else c.ctypes.data


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

    def _chain(self, family, head, n, harvest_options, dio_options, outs, cheaptrick_options=None, d4c_options=None,
               device=False, rows=None):
        """Calls the analysis chain world_b200_<family> whose variant fits the per-utterance option lists given
        (_options: Harvest, _dio_options: DIO, _spectral_options: CheapTrick / D4C, with either F0 list).  head: the
        arguments between the handle and the option arrays; outs: those after them.  rows: the (spectrogram,
        aperiodicity) arrays of a full-row chain, whose _spectral_options variant takes their last dimension as the
        row_stride after f0_stride.  device: the chain is enqueued on torch's current stream."""
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        if cheaptrick_options is not None or d4c_options is not None:
            ct = None if cheaptrick_options is None else _option_array(CheapTrickOption, cheaptrick_options, n)
            d4 = None if d4c_options is None else _option_array(D4COption, d4c_options, n)
            suffix, arrays = "_spectral_options", (per_utt, per_dio, ct, d4)
            if rows is not None:
                outs = (*outs[:3], _row_stride(*rows), *outs[3:])
        elif per_utt is not None:
            suffix, arrays = "_options", (per_utt,)
        elif per_dio is not None:
            suffix, arrays = "_dio_options", (per_dio,)
        else:
            suffix, arrays = "", ()
        if device:
            self._use_current_stream()
        self._check(getattr(self.lib, f"world_b200_{family}{suffix}")(self._h, *head, *arrays, *outs))

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
        out = self._zeros(x, tuple(f0.shape))
        return self._stage("stonemask_batch", x, fs, time_axis, f0, x_lengths, f0_lengths, (), out)

    def cheaptrick(self, x, fs, time_axis, f0, option: CheapTrickOption | None = None, x_lengths=None,
                   f0_lengths=None, out=None):
        """option: one CheapTrickOption for the batch, or a list of one per utterance (each speaker's fft_size from
        its own F0 floor).  With a list the rows are [n, L, max fft_size / 2 + 1] (or out's last dimension): the
        first fft_size / 2 + 1 values of utterance u's rows are written, the rest are left as they are."""
        if out is None:
            sizes = ([o.fft_size for o in option] if isinstance(option, (list, tuple))
                     else [(option or self.cheaptrick_option(fs)).fft_size])
            out = self._zeros(x, (x.shape[0], f0.shape[1], max(sizes or [0]) // 2 + 1))
        return self._cheaptrick(False, x, fs, time_axis, f0, option, x_lengths, f0_lengths, out.shape[-1], out)

    def d4c(self, x, fs, time_axis, f0, fft_size, option: D4COption | None = None, x_lengths=None,
            f0_lengths=None, out=None):
        """fft_size / option: one for the batch, or either as a list of one per utterance; then the rows are
        [n, L, max fft_size / 2 + 1] (or out's last dimension) and utterance u writes fft_size[u] / 2 + 1 of each."""
        if out is None:
            sizes = list(fft_size) if isinstance(fft_size, (list, tuple)) else [int(fft_size)] * x.shape[0]
            out = self._zeros(x, (x.shape[0], f0.shape[1], max(sizes or [0]) // 2 + 1))
        return self._d4c(False, x, fs, time_axis, f0, fft_size, option, x_lengths, f0_lengths, out)

    def cheaptrick_coded(self, x, fs, time_axis, f0, number_of_dimensions, option: CheapTrickOption | None = None,
                         x_lengths=None, f0_lengths=None):
        """CheapTrick + CodeSpectralEnvelope in one kernel per frame -> [n, L, number_of_dimensions].  option may be
        a list of one CheapTrickOption per utterance (each coded at its own fft_size)."""
        out = self._zeros(x, (x.shape[0], f0.shape[1], number_of_dimensions))
        return self._cheaptrick(True, x, fs, time_axis, f0, option, x_lengths, f0_lengths, number_of_dimensions, out)

    def d4c_coded(self, x, fs, time_axis, f0, fft_size, option: D4COption | None = None, x_lengths=None,
                  f0_lengths=None):
        """D4C + CodeAperiodicity in one kernel per frame -> [n, L, GetNumberOfAperiodicities(fs)].  fft_size and
        option may be lists of one per utterance."""
        out = self._zeros(x, (x.shape[0], f0.shape[1], max(1, self.number_of_aperiodicities(fs))))
        return self._d4c(True, x, fs, time_axis, f0, fft_size, option, x_lengths, f0_lengths, out)

    def _stage(self, entry, x, fs, time_axis, f0, x_lengths, f0_lengths, options, out):
        """Calls the stage entry point world_b200_<entry> on the rows x / time_axis / f0 with options (the arguments
        between f0_stride and the output) into out, enqueued on the current stream; returns out."""
        n, stride = x.shape
        xl, k1 = _int_array(x_lengths, n)
        fl, k2 = _int_array(f0_lengths, n)
        self._use_current_stream()
        self._check(getattr(self.lib, f"world_b200_{entry}")(self._h, _ptr(x), n, stride, xl, fs, _ptr(time_axis),
                                                             _ptr(f0), fl, f0.shape[1], *options, _ptr(out)))
        return out

    def _cheaptrick(self, coded, x, fs, time_axis, f0, option, x_lengths, f0_lengths, width, out):
        """CheapTrick into full or coded rows.  option: one CheapTrickOption (None: the default at fs) or a list of one
        per utterance.  width: number_of_dimensions (coded), or the row_stride of a list's full rows."""
        if isinstance(option, (list, tuple)):
            suffix, options = "_options", (_option_array(CheapTrickOption, option, x.shape[0]), width)
        else:
            suffix, options = "", (C.byref(option or self.cheaptrick_option(fs)),) + ((width,) if coded else ())
        entry = f"cheaptrick{'_coded' if coded else ''}_batch{suffix}"
        return self._stage(entry, x, fs, time_axis, f0, x_lengths, f0_lengths, options, out)

    def _d4c(self, coded, x, fs, time_axis, f0, fft_size, option, x_lengths, f0_lengths, out):
        """D4C into full or coded rows; fft_size / option: one for the batch, or either as a list of one per
        utterance (full rows then take out's last dimension as their row_stride)."""
        if isinstance(fft_size, (list, tuple)) or isinstance(option, (list, tuple)):
            sizes, opts = self._d4c_options(fft_size, option, x.shape[0])
            suffix, options = "_options", (sizes, opts) + (() if coded else (out.shape[-1],))
        else:
            suffix, options = "", (fft_size, C.byref(option or self.d4c_option()))
        entry = f"d4c{'_coded' if coded else ''}_batch{suffix}"
        return self._stage(entry, x, fs, time_axis, f0, x_lengths, f0_lengths, options, out)

    def _d4c_options(self, fft_size, option, n):
        """Per-utterance D4C arguments as ctypes arrays: a scalar fft_size or option applies to every utterance."""
        sizes = list(fft_size) if isinstance(fft_size, (list, tuple)) else [int(fft_size)] * n
        if len(sizes) != n:
            raise ValueError(f"{len(sizes)} fft sizes for {n} utterances")
        opts = option if isinstance(option, (list, tuple)) else [option or self.d4c_option()] * n
        return (C.c_int * n)(*sizes), _option_array(D4COption, opts, n)

    def synthesis(self, f0, spectrogram, aperiodicity, fft_size, frame_period, fs, y_length, f0_lengths=None,
                  y_lengths=None):
        """Batched Synthesis(): f0 [n, L], spectrogram / aperiodicity [n, L, bins] -> y [n, y_length].  fft_size may
        be a sequence of one size per utterance (world_b200_synthesis_batch_options): the rows are then
        [n, L, row_stride], as cheaptrick / d4c with per-utterance options write them, and utterance u reads the first
        fft_size[u] / 2 + 1 values of each."""
        n = f0.shape[0]
        y = self._zeros(f0, (n, y_length))
        fl, k1 = _int_array(f0_lengths, n)
        yl, k2 = _int_array(y_lengths, n)
        sizes = _fft_sizes(fft_size, n)
        self._use_current_stream()
        if sizes is not None:
            self._check(self.lib.world_b200_synthesis_batch_options(
                self._h, _ptr(f0), fl, n, f0.shape[1], _ptr(spectrogram), _ptr(aperiodicity),
                int(spectrogram.shape[-1]), sizes, frame_period, fs, yl, y_length, _ptr(y)))
            return y
        self._check(self.lib.world_b200_synthesis_batch(self._h, _ptr(f0), fl, n, f0.shape[1], _ptr(spectrogram),
                                                        _ptr(aperiodicity), fft_size, frame_period, fs, yl, y_length,
                                                        _ptr(y)))
        return y

    def synthesis_coded(self, f0, coded_spectral_envelope, coded_aperiodicity, fft_size, frame_period, fs, y_length,
                        f0_lengths=None, y_lengths=None, dtype=None, f0_scale=None, spectral_ratio=None):
        """Batched Synthesis() from coded rows: f0 [n, L], coded_spectral_envelope [n, L, number_of_dimensions],
        coded_aperiodicity [n, L, GetNumberOfAperiodicities(fs)] -> y [n, y_length].  The rows are decoded chunk by
        chunk inside the call; the output equals decode_spectral_envelope + decode_aperiodicity + synthesis bit for
        bit.  coded_aperiodicity may be None below 12 kHz (no bands).  dtype: float64 (default) for the waveform, or
        int16 for its 16-bit PCM, quantised as wavwrite does by the overlap-add kernel itself.
        f0_scale / spectral_ratio (one factor, or one per utterance): synthesise the voice changed as modify() changes
        it, without touching the inputs (world_b200_synthesis_coded_batch_modified); the output equals decode +
        modify + synthesis bit for bit.
        fft_size may be a sequence of one size per utterance (world_b200_synthesis_coded_batch_options): each utterance
        is decoded and synthesised at its own size."""
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
        sizes = _fft_sizes(fft_size, n)
        self._use_current_stream()
        entry = (self.lib.world_b200_synthesis_coded_batch_modified if sizes is None
                 else self.lib.world_b200_synthesis_coded_batch_options)
        self._check(entry(
            self._h, _ptr(f0), fl, n, f0.shape[1], _ptr(coded_spectral_envelope),
            int(coded_spectral_envelope.shape[-1]), _ptr(coded_aperiodicity), fft_size if sizes is None else sizes,
            frame_period, fs, yl, y_length, _factors(f0_scale, n, "f0_scale"),
            _factors(spectral_ratio, n, "spectral_ratio"), 16 if pcm16 else 0, _ptr(y)))
        return y

    def modify(self, f0, spectrogram, fs, fft_size, f0_scale=None, spectral_ratio=None, f0_lengths=None):
        """F0 scaling and formant shift in place (world_b200_modify_batch, the reference demo's ParameterModification):
        f0 [n, L] *= f0_scale, and each envelope row [n, L, fft_size/2+1] is stretched along frequency by
        spectral_ratio.  Either factor may be one number for every utterance, a sequence of one per utterance, or None
        to leave that array alone (it may then be None too).  fft_size may be a sequence of one size per utterance
        (world_b200_modify_batch_options): the rows are then [n, L, row_stride] and utterance u's envelope is the first
        fft_size[u] / 2 + 1 values of each.  Returns (f0, spectrogram)."""
        rows = f0 if f0 is not None else spectrogram
        n, L = int(rows.shape[0]), int(rows.shape[1])
        fl, k1 = _int_array(f0_lengths, n)
        sizes = _fft_sizes(fft_size, n)
        self._use_current_stream()
        if sizes is not None:
            row = int(spectrogram.shape[-1]) if spectrogram is not None else 0
            self._check(self.lib.world_b200_modify_batch_options(
                self._h, _ptr(f0), fl, n, L, _ptr(spectrogram), row, sizes, fs, _factors(f0_scale, n, "f0_scale"),
                _factors(spectral_ratio, n, "spectral_ratio")))
            return f0, spectrogram
        self._check(self.lib.world_b200_modify_batch(self._h, _ptr(f0), fl, n, L, _ptr(spectrogram), fft_size, fs,
                                                     _factors(f0_scale, n, "f0_scale"),
                                                     _factors(spectral_ratio, n, "spectral_ratio")))
        return f0, spectrogram

    def synthesis_coded_host(self, f0, coded_sp, coded_ap, fft_size, frame_period, fs, y_length, nbit=16,
                             f0_lengths=None, y_lengths=None, out=None, f0_scale=None, spectral_ratio=None):
        """synthesis_coded for HOST arrays (numpy arrays or CPU tensors, float64): upload, synthesis and download are
        pipelined over utterance chunks (world_b200_synthesis_coded_host).  Returns y [n, y_length] as a numpy array,
        int16 for nbit 16 or float64 for nbit 0, whole rows (samples beyond an utterance's y_length are 0).  out: a
        host array of that shape and dtype to write into (a pinned one lets the downloads overlap the kernels).
        coded_ap may be None below 12 kHz (no bands).  f0_scale / spectral_ratio as in synthesis_coded
        (world_b200_synthesis_coded_host_modified).  fft_size may be a sequence of one size per utterance
        (world_b200_synthesis_coded_host_options)."""
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
        sizes = _fft_sizes(fft_size, n)
        entry = (self.lib.world_b200_synthesis_coded_host_modified if sizes is None
                 else self.lib.world_b200_synthesis_coded_host_options)
        self._check(entry(
            self._h, _ptr(f0), fl, n, f0.shape[1], _ptr(coded_sp), int(coded_sp.shape[-1]), _ptr(coded_ap),
            fft_size if sizes is None else sizes, frame_period, fs, yl, y_length, _factors(f0_scale, n, "f0_scale"),
            _factors(spectral_ratio, n, "spectral_ratio"), nbit, _ptr(y)))
        return y

    def analysis_option(self, fs, f0_method=F0_HARVEST) -> AnalysisOption:
        o = AnalysisOption()
        self.lib.world_b200_default_analysis_option(fs, f0_method, C.byref(o))
        return o

    def analyze_batch(self, x, fs, option: AnalysisOption, x_lengths=None, time_axis=None, f0=None,
                      spectrogram=None, aperiodicity=None, harvest_options=None, dio_options=None,
                      cheaptrick_options=None, d4c_options=None):
        """Whole chain on DEVICE arrays in one call (two internal streams); returns (t, f0, sp, ap, frame counts).
        harvest_options: a list of one HarvestOption per utterance (Harvest with a per-utterance F0 range);
        dio_options: a list of one DioOption per utterance (DIO + StoneMask with a per-utterance F0 range).
        cheaptrick_options / d4c_options: a list of one CheapTrickOption / D4COption per utterance
        (world_b200_analyze_batch_spectral_options; D4C runs at each utterance's CheapTrick fft_size).  The rows are
        then [n, L, row_stride] with row_stride the last dimension of spectrogram (allocated as max fft_size // 2 + 1
        when None), and utterance u writes the first fft_size[u] // 2 + 1 values of each of its frames."""
        n, stride = x.shape
        frame_period = _frame_period(option)
        f_stride, fl = self._f0_stride(fs, x, x_lengths, frame_period)
        bins = _full_bins(option, cheaptrick_options)
        if time_axis is None:
            time_axis = self._zeros(x, (n, f_stride))
        if f0 is None:
            f0 = self._zeros(x, (n, f_stride))
        if spectrogram is None:
            spectrogram = self._zeros(x, (n, f_stride, bins))
        if aperiodicity is None:
            aperiodicity = self._zeros(x, (n, f_stride, bins))
        xl, keep = _int_array(x_lengths, n)
        self._chain("analyze_batch", (_ptr(x), n, stride, xl, fs, C.byref(option)), n, harvest_options, dio_options,
                    (_ptr(time_axis), _ptr(f0), time_axis.shape[1], _ptr(spectrogram), _ptr(aperiodicity)),
                    cheaptrick_options=cheaptrick_options, d4c_options=d4c_options, device=True,
                    rows=(spectrogram, aperiodicity))
        return time_axis, f0, spectrogram, aperiodicity, fl

    # -- packed batches: utterances back to back, utterance u = samples [x_offsets[u], x_offsets[u + 1]) --------
    def packed_frames(self, fs, x_offsets, frame_period=5.0):
        """The frame offsets of a packed batch (numpy int64, n + 1): utterance u's frames are rows
        [f[u], f[u + 1]) of the packed outputs, f[n] = F in all."""
        import numpy as np
        n, xo = _offsets(x_offsets)
        f = (C.c_longlong * (n + 1))()
        rc = self.lib.world_b200_packed_frames(fs, n, xo, frame_period, f)
        if rc:
            raise WorldError(f"world_b200_packed_frames: bad x_offsets or arguments (code {rc})")
        return np.array(f[:], dtype=np.int64)

    def _packed(self, name, x, head, x_offsets, fs, option, mid, widths, outs, harvest_options, dio_options,
                cheaptrick_options, d4c_options, device):
        """Calls world_b200_<name> on a packed batch: head = the arguments before n_utts, mid = those between the
        option arrays and the output arrays; outs = (time_axis, f0, spectrogram, aperiodicity), each allocated when
        None with F frames of widths (0: [F]); full rows pass row_stride (widths' row) after f0.  Returns the outputs
        and the frame offsets."""
        import numpy as np
        n, xo = _offsets(x_offsets)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        ct = None if cheaptrick_options is None else _option_array(CheapTrickOption, cheaptrick_options, n)
        d4 = None if d4c_options is None else _option_array(D4COption, d4c_options, n)
        outs = list(outs)
        for i, w in enumerate(widths):
            if outs[i] is None:
                F = int(self.packed_frames(fs, x_offsets, _frame_period(option))[-1])
                shape = (F, w) if w else (F,)
                outs[i] = self._zeros(x, shape) if device else np.zeros(shape)
        f = (C.c_longlong * (n + 1))()
        args = [_ptr(outs[0]), _ptr(outs[1])]
        if mid is None:   # full rows: the row_stride of the arrays
            args.append(_row_stride(outs[2], outs[3]))
        args += [_ptr(outs[2]), _ptr(outs[3]), f]
        if device:
            self._use_current_stream()
        self._check(getattr(self.lib, f"world_b200_{name}")(self._h, _ptr(x), *head, n, xo, fs, C.byref(option),
                                                             per_utt, per_dio, ct, d4, *([] if mid is None else mid),
                                                             *args))
        return (*outs, np.array(f[:], dtype=np.int64))

    def analyze_packed(self, x, x_offsets, fs, option: AnalysisOption, harvest_options=None, dio_options=None,
                       cheaptrick_options=None, d4c_options=None, row_stride=0, time_axis=None, f0=None,
                       spectrogram=None, aperiodicity=None):
        """analyze_batch on a PACKED batch of DEVICE float64 samples (world_b200_analyze_packed): x holds the
        utterances back to back, utterance u being samples [x_offsets[u], x_offsets[u + 1]) (x_offsets: n + 1
        offsets, a list, numpy array or CPU tensor).  Returns (time_axis [F], f0 [F], spectrogram [F, W],
        aperiodicity [F, W], f_offsets [n + 1]): utterance u's frames are rows [f_offsets[u], f_offsets[u + 1]).
        W = row_stride, or the largest fft_size // 2 + 1 when 0; given arrays set W by their last dimension.  Each
        utterance's values equal analyze_batch's, bit for bit; the rest of each row is not written."""
        W = row_stride or (_row_stride(spectrogram, aperiodicity) if spectrogram is not None or aperiodicity is not None
                           else _full_bins(option, cheaptrick_options))
        return self._packed("analyze_packed", x, (), x_offsets, fs, option, None, (0, 0, W, W),
                            (time_axis, f0, spectrogram, aperiodicity), harvest_options, dio_options,
                            cheaptrick_options, d4c_options, device=True)

    def analyze_host_packed(self, x_host, x_offsets, fs, option: AnalysisOption, harvest_options=None,
                            dio_options=None, cheaptrick_options=None, d4c_options=None, row_stride=0, time_axis=None,
                            f0=None, spectrogram=None, aperiodicity=None):
        """analyze_packed on HOST arrays (world_b200_analyze_host_packed), outputs allocated with numpy when None;
        full rows read 0 past each utterance's fft_size // 2 + 1."""
        W = row_stride or (_row_stride(spectrogram, aperiodicity) if spectrogram is not None or aperiodicity is not None
                           else _full_bins(option, cheaptrick_options))
        return self._packed("analyze_host_packed", x_host, (), x_offsets, fs, option, None, (0, 0, W, W),
                            (time_axis, f0, spectrogram, aperiodicity), harvest_options, dio_options,
                            cheaptrick_options, d4c_options, device=False)

    def analyze_coded_packed(self, x, nbit, x_offsets, fs, option: AnalysisOption, number_of_dimensions,
                             harvest_options=None, dio_options=None, cheaptrick_options=None, d4c_options=None,
                             time_axis=None, f0=None, coded_sp=None, coded_ap=None):
        """analyze_coded_batch on a PACKED batch (world_b200_analyze_coded_packed): x holds float64 samples (nbit 0)
        or nbit-bit PCM back to back, sample offsets as for analyze_packed.  Returns (time_axis [F], f0 [F],
        coded_sp [F, number_of_dimensions], coded_ap [F, max(1, GetNumberOfAperiodicities(fs))], f_offsets)."""
        n_ap = max(1, self.number_of_aperiodicities(fs))
        return self._packed("analyze_coded_packed", x, (nbit,), x_offsets, fs, option, (number_of_dimensions,),
                            (0, 0, number_of_dimensions, n_ap), (time_axis, f0, coded_sp, coded_ap), harvest_options,
                            dio_options, cheaptrick_options, d4c_options, device=True)

    def analyze_coded_host_packed(self, x_host, nbit, x_offsets, fs, option: AnalysisOption, number_of_dimensions,
                                  harvest_options=None, dio_options=None, cheaptrick_options=None, d4c_options=None,
                                  time_axis=None, f0=None, coded_sp=None, coded_ap=None):
        """analyze_coded_packed on HOST arrays (world_b200_analyze_coded_host_packed)."""
        n_ap = max(1, self.number_of_aperiodicities(fs))
        return self._packed("analyze_coded_host_packed", x_host, (nbit,), x_offsets, fs, option,
                            (number_of_dimensions,), (0, 0, number_of_dimensions, n_ap),
                            (time_axis, f0, coded_sp, coded_ap), harvest_options, dio_options, cheaptrick_options,
                            d4c_options, device=False)

    # -- the way back on packed rows: utterance u = frames [f_offsets[u], f_offsets[u + 1]) and samples
    #    [y_offsets[u], y_offsets[u + 1]) ----------------------------------------------------------------------------
    def _packed_way_back(self, f_offsets, y_offsets, fft_size):
        """(n, f_offsets, y_offsets as ctypes int64 arrays, Y, per-utterance fft sizes as a ctypes int array)."""
        n, fo = _offsets(f_offsets)
        ny, yo = _offsets(y_offsets)
        if ny != n:
            raise ValueError(f"{n + 1} f_offsets but {ny + 1} y_offsets")
        sizes = _fft_sizes(fft_size, n)
        if sizes is None:
            sizes = (C.c_int * max(n, 1))(*([int(fft_size)] * n))
        return n, fo, yo, int(yo[n]), sizes

    def _packed_y(self, like, Y, pcm16):
        if self.xp == "torch":
            dtype = self.torch.int16 if pcm16 else self.torch.float64
            return self.torch.zeros((Y,), dtype=dtype, device=like.device)
        import numpy as np
        return np.zeros((Y,), dtype=np.int16 if pcm16 else np.float64)

    def synthesis_packed(self, f0, spectrogram, aperiodicity, f_offsets, fft_size, frame_period, fs, y_offsets,
                         y=None):
        """synthesis on PACKED rows of DEVICE arrays (world_b200_synthesis_packed): f0 [F], spectrogram / aperiodicity
        [F, W] (W >= every fft_size // 2 + 1, as analyze_packed writes them), utterance u being frames
        [f_offsets[u], f_offsets[u + 1]).  Returns y [Y] (float64), utterance u being samples
        [y_offsets[u], y_offsets[u + 1]); offsets as analyze_packed takes them.  fft_size: one int, or one per
        utterance.  Each utterance's samples equal synthesis()'s with the same sizes, bit for bit."""
        n, fo, yo, Y, sizes = self._packed_way_back(f_offsets, y_offsets, fft_size)
        if y is None:
            y = self._packed_y(f0, Y, False)
        self._use_current_stream()
        self._check(self.lib.world_b200_synthesis_packed(
            self._h, _ptr(f0), n, fo, _ptr(spectrogram), _ptr(aperiodicity), int(spectrogram.shape[-1]), sizes,
            frame_period, fs, yo, _ptr(y)))
        return y

    def synthesis_coded_packed(self, f0, coded_spectral_envelope, coded_aperiodicity, f_offsets, fft_size,
                               frame_period, fs, y_offsets, dtype=None, f0_scale=None, spectral_ratio=None, y=None):
        """synthesis_coded on PACKED rows of DEVICE arrays (world_b200_synthesis_coded_packed): f0 [F],
        coded_spectral_envelope [F, number_of_dimensions], coded_aperiodicity [F, GetNumberOfAperiodicities(fs)] (may
        be None below 12 kHz).  Returns y [Y], float64 or (dtype int16) 16-bit PCM.  f0_scale / spectral_ratio as in
        synthesis_coded."""
        pcm16 = _pcm16(dtype)
        n, fo, yo, Y, sizes = self._packed_way_back(f_offsets, y_offsets, fft_size)
        if y is None:
            y = self._packed_y(f0, Y, pcm16)
        self._use_current_stream()
        self._check(self.lib.world_b200_synthesis_coded_packed(
            self._h, _ptr(f0), n, fo, _ptr(coded_spectral_envelope), int(coded_spectral_envelope.shape[-1]),
            _ptr(coded_aperiodicity), sizes, frame_period, fs, yo, _factors(f0_scale, n, "f0_scale"),
            _factors(spectral_ratio, n, "spectral_ratio"), 16 if pcm16 else 0, _ptr(y)))
        return y

    def synthesis_coded_host_packed(self, f0, coded_sp, coded_ap, f_offsets, fft_size, frame_period, fs, y_offsets,
                                    nbit=16, out=None, f0_scale=None, spectral_ratio=None):
        """synthesis_coded_packed for HOST arrays (numpy arrays or CPU tensors, float64), pipelined over chunks of
        utterances (world_b200_synthesis_coded_host_packed).  Returns y [Y] as a numpy array, int16 for nbit 16 or
        float64 for nbit 0.  out: a contiguous host array of that shape and dtype to write into (pinned, the downloads
        overlap the kernels)."""
        import numpy as np

        def host(a):
            if a is None:
                return None
            if hasattr(a, "numpy"):
                a = a.detach().numpy()
            return np.ascontiguousarray(a, dtype=np.float64)

        f0, coded_sp, coded_ap = host(f0), host(coded_sp), host(coded_ap)
        n, fo, yo, Y, sizes = self._packed_way_back(f_offsets, y_offsets, fft_size)
        dt = np.int16 if nbit == 16 else np.float64
        if out is None:
            out = np.empty((Y,), dtype=dt)
        y = out.numpy() if hasattr(out, "numpy") else out
        if nbit in (0, 16) and (y.shape != (Y,) or y.dtype != dt or not y.flags.c_contiguous):
            raise ValueError(f"out: a contiguous [{Y}] {np.dtype(dt).name} host array")
        self._check(self.lib.world_b200_synthesis_coded_host_packed(
            self._h, _ptr(f0), n, fo, _ptr(coded_sp), int(coded_sp.shape[-1]), _ptr(coded_ap), sizes, frame_period,
            fs, yo, _factors(f0_scale, n, "f0_scale"), _factors(spectral_ratio, n, "spectral_ratio"), nbit, _ptr(y)))
        return y

    def modify_packed(self, f0, spectrogram, f_offsets, fs, fft_size=None, f0_scale=None, spectral_ratio=None):
        """modify on PACKED rows in place (world_b200_modify_packed): f0 [F], spectrogram [F, W] (W >= every
        fft_size // 2 + 1), utterance u being frames [f_offsets[u], f_offsets[u + 1]).  fft_size (one int or one per
        utterance) is needed with spectral_ratio.  Returns (f0, spectrogram)."""
        n, fo = _offsets(f_offsets)
        sizes = None
        if fft_size is not None:
            sizes = _fft_sizes(fft_size, n)
            if sizes is None:
                sizes = (C.c_int * max(n, 1))(*([int(fft_size)] * n))
        row = int(spectrogram.shape[-1]) if spectrogram is not None else 0
        self._use_current_stream()
        self._check(self.lib.world_b200_modify_packed(
            self._h, _ptr(f0), n, fo, _ptr(spectrogram), row, sizes, fs, _factors(f0_scale, n, "f0_scale"),
            _factors(spectral_ratio, n, "spectral_ratio")))
        return f0, spectrogram

    # -- pitch and formant curves: one f0 factor and one spectral ratio per frame -----------------------------------
    def modify_curves(self, f0, spectrogram, fs, fft_size, f0_curve=None, spectral_ratio_curve=None, f0_lengths=None):
        """modify with one factor per FRAME in place (world_b200_modify_curves): f0 [n, L] *= f0_curve [n, L], and
        frame i of utterance u's envelope [n, L, W] is stretched by spectral_ratio_curve[u, i] at fft_size (one int, or
        one per utterance; W >= every fft_size // 2 + 1).  The curves are arrays on the rows' device (either may be
        None, which leaves that half alone).  The call checks every frame of the curves on the device before it
        modifies anything, and so synchronises the stream once.  Returns (f0, spectrogram)."""
        rows = f0 if f0 is not None else spectrogram
        n, L = int(rows.shape[0]), int(rows.shape[1])
        fl, k1 = _int_array(f0_lengths, n)
        sizes = _curve_sizes(fft_size, n)
        row = int(spectrogram.shape[-1]) if spectrogram is not None else 0
        self._use_current_stream()
        self._check(self.lib.world_b200_modify_curves(self._h, _ptr(f0), fl, n, L, _ptr(spectrogram), row, sizes, fs,
                                                      _curve(f0_curve), _curve(spectral_ratio_curve)))
        return f0, spectrogram

    def modify_curves_packed(self, f0, spectrogram, f_offsets, fs, fft_size=None, f0_curve=None,
                             spectral_ratio_curve=None):
        """modify_curves on PACKED rows in place (world_b200_modify_curves_packed): f0 [F], spectrogram [F, W] and the
        curves [F] on the rows' device, utterance u being frames [f_offsets[u], f_offsets[u + 1]).  fft_size (one int
        or one per utterance) is needed with spectral_ratio_curve.  Returns (f0, spectrogram)."""
        n, fo = _offsets(f_offsets)
        sizes = None if fft_size is None else _curve_sizes(fft_size, n)
        row = int(spectrogram.shape[-1]) if spectrogram is not None else 0
        self._use_current_stream()
        self._check(self.lib.world_b200_modify_curves_packed(self._h, _ptr(f0), n, fo, _ptr(spectrogram), row, sizes,
                                                             fs, _curve(f0_curve), _curve(spectral_ratio_curve)))
        return f0, spectrogram

    # -- the stage calls on packed batches: utterance u = samples [x_offsets[u], x_offsets[u + 1]) of x and frames
    #    [f_offsets[u], f_offsets[u + 1]) of time_axis, f0 and the rows ------------------------------------------------
    def _stage_packed(self, entry, x, x_offsets, fs, time_axis, f0, f_offsets, options, out):
        """Calls world_b200_<entry> on packed DEVICE arrays with options (the arguments between f_offsets and the
        output) into out, enqueued on the current stream; returns out."""
        n, xo = _offsets(x_offsets)
        nf, fo = _offsets(f_offsets)
        if nf != n:
            raise ValueError(f"{n + 1} x_offsets but {nf + 1} f_offsets")
        self._use_current_stream()
        self._check(getattr(self.lib, f"world_b200_{entry}")(self._h, _ptr(x), n, xo, fs, _ptr(time_axis), _ptr(f0),
                                                             fo, *options, _ptr(out)))
        return out

    def _packed_options(self, cls, option, n, default):
        """One option (None: default()) for every utterance, or a list of n -> a ctypes array of n."""
        if option is None or isinstance(option, cls):
            option = [option or default()] * n
        return _option_array(cls, option, n)

    def _packed_sizes(self, fft_size, n):
        sizes = _fft_sizes(fft_size, n)
        return sizes if sizes is not None else (C.c_int * max(n, 1))(*([int(fft_size)] * n))

    def _packed_rows(self, like, f_offsets, width, out):
        """out, or zeros [F, width] with F = f_offsets[-1]."""
        if out is not None:
            return out
        n, fo = _offsets(f_offsets)
        return self._zeros(like, (int(fo[n]), width))

    def stonemask_packed(self, x, x_offsets, fs, time_axis, f0, f_offsets, out=None):
        """stonemask on a PACKED batch of DEVICE arrays (world_b200_stonemask_packed): x holds the utterances back to
        back (x_offsets: n + 1 sample offsets), time_axis / f0 their frames back to back (f_offsets: n + 1 frame
        offsets, the caller's own or analyze_packed's).  Offsets may be a list, numpy array or CPU tensor.  Returns the
        refined f0 [F] (out, which may be f0 itself).  Each utterance's values equal stonemask()'s bit for bit."""
        if out is None:
            out = self._zeros(f0, tuple(f0.shape))
        return self._stage_packed("stonemask_packed", x, x_offsets, fs, time_axis, f0, f_offsets, (), out)

    def _cheaptrick_packed(self, coded, x, x_offsets, fs, time_axis, f0, f_offsets, option, width, out):
        n = len(x_offsets) - 1
        opts = self._packed_options(CheapTrickOption, option, n, lambda: self.cheaptrick_option(fs))
        if out is None:
            if not coded:
                width = width or max([o.fft_size for o in opts] or [0]) // 2 + 1
            out = self._packed_rows(f0, f_offsets, width, None)
        elif not coded:
            width = int(out.shape[-1])
        entry = "cheaptrick_coded_packed" if coded else "cheaptrick_packed"
        return self._stage_packed(entry, x, x_offsets, fs, time_axis, f0, f_offsets, (opts, width), out)

    def cheaptrick_packed(self, x, x_offsets, fs, time_axis, f0, f_offsets, option=None, row_stride=0, out=None):
        """cheaptrick on a PACKED batch (world_b200_cheaptrick_packed), arrays and offsets as stonemask_packed.
        option: one CheapTrickOption for every utterance (None: the default at fs) or a list of one per utterance.
        Returns the spectrogram [F, W]: W = out's last dimension, or row_stride, or the largest fft_size // 2 + 1.
        Utterance u writes the first fft_size[u] // 2 + 1 values of each of its rows, equal to cheaptrick()'s."""
        return self._cheaptrick_packed(False, x, x_offsets, fs, time_axis, f0, f_offsets, option, row_stride, out)

    def cheaptrick_coded_packed(self, x, x_offsets, fs, time_axis, f0, f_offsets, number_of_dimensions, option=None,
                                out=None):
        """cheaptrick_coded on a PACKED batch (world_b200_cheaptrick_coded_packed) -> [F, number_of_dimensions]."""
        return self._cheaptrick_packed(True, x, x_offsets, fs, time_axis, f0, f_offsets, option,
                                       number_of_dimensions, out)

    def _d4c_packed(self, coded, x, x_offsets, fs, time_axis, f0, f_offsets, fft_size, option, row_stride, out):
        n = len(x_offsets) - 1
        sizes = self._packed_sizes(fft_size, n)
        opts = None if option is None else self._packed_options(D4COption, option, n, self.d4c_option)
        if coded:
            out = self._packed_rows(f0, f_offsets, max(1, self.number_of_aperiodicities(fs)), out)
            options = (sizes, opts)
        else:
            out = self._packed_rows(f0, f_offsets, row_stride or max(list(sizes)[:n] or [0]) // 2 + 1, out)
            options = (sizes, opts, int(out.shape[-1]))
        entry = "d4c_coded_packed" if coded else "d4c_packed"
        return self._stage_packed(entry, x, x_offsets, fs, time_axis, f0, f_offsets, options, out)

    def d4c_packed(self, x, x_offsets, fs, time_axis, f0, f_offsets, fft_size, option=None, row_stride=0, out=None):
        """d4c on a PACKED batch (world_b200_d4c_packed), arrays and offsets as stonemask_packed.  fft_size: one int
        or one per utterance (its CheapTrick size); option: one D4COption, a list of one per utterance, or None
        (InitializeD4COption).  Returns the aperiodicity [F, W], W as in cheaptrick_packed."""
        return self._d4c_packed(False, x, x_offsets, fs, time_axis, f0, f_offsets, fft_size, option, row_stride, out)

    def d4c_coded_packed(self, x, x_offsets, fs, time_axis, f0, f_offsets, fft_size, option=None, out=None):
        """d4c_coded on a PACKED batch (world_b200_d4c_coded_packed) -> [F, max(1, GetNumberOfAperiodicities(fs))]
        (nothing is written below 12 kHz)."""
        return self._d4c_packed(True, x, x_offsets, fs, time_axis, f0, f_offsets, fft_size, option, 0, out)

    def _codec_packed(self, entry, src, f_offsets, full_rows, fs, fft_size, dims, width, out):
        """world_b200_<entry> between full rows [F, W] and coded rows [F, dims]; full_rows: the full-row array (the
        input when coding, the output when decoding), whose last dimension is the row_stride."""
        n, fo = _offsets(f_offsets)
        sizes = self._packed_sizes(fft_size, n)
        if out is None:
            out = self._packed_rows(src, f_offsets, width, None)
        row = int((src if full_rows == "in" else out).shape[-1])
        args = [self._h, _ptr(src), n, fo, row, sizes, fs] + ([] if dims is None else [dims])
        self._use_current_stream()
        self._check(getattr(self.lib, f"world_b200_{entry}")(*args, _ptr(out)))
        return out

    def code_spectral_envelope_packed(self, spectrogram, f_offsets, fs, fft_size, number_of_dimensions, out=None):
        """code_spectral_envelope on PACKED rows (world_b200_code_spectral_envelope_packed): spectrogram [F, W] (W >=
        every fft_size // 2 + 1), utterance u being frames [f_offsets[u], f_offsets[u + 1]) at fft_size (one int or
        one per utterance) -> [F, number_of_dimensions]."""
        return self._codec_packed("code_spectral_envelope_packed", spectrogram, f_offsets, "in", fs, fft_size,
                                  number_of_dimensions, number_of_dimensions, out)

    def decode_spectral_envelope_packed(self, coded, f_offsets, fs, fft_size, number_of_dimensions, row_stride=0,
                                        out=None):
        """decode_spectral_envelope on PACKED rows -> [F, W] (W: out's last dimension, or row_stride, or the largest
        fft_size // 2 + 1); utterance u writes the first fft_size[u] // 2 + 1 values of each row."""
        n = len(f_offsets) - 1
        W = row_stride or max(list(self._packed_sizes(fft_size, n))[:n] or [0]) // 2 + 1
        return self._codec_packed("decode_spectral_envelope_packed", coded, f_offsets, "out", fs, fft_size,
                                  number_of_dimensions, W, out)

    def code_aperiodicity_packed(self, aperiodicity, f_offsets, fs, fft_size, out=None):
        """code_aperiodicity on PACKED rows -> [F, max(1, GetNumberOfAperiodicities(fs))]."""
        return self._codec_packed("code_aperiodicity_packed", aperiodicity, f_offsets, "in", fs, fft_size, None,
                                  max(1, self.number_of_aperiodicities(fs)), out)

    def decode_aperiodicity_packed(self, coded, f_offsets, fs, fft_size, row_stride=0, out=None):
        """decode_aperiodicity on PACKED rows -> [F, W], W as in decode_spectral_envelope_packed."""
        n = len(f_offsets) - 1
        W = row_stride or max(list(self._packed_sizes(fft_size, n))[:n] or [0]) // 2 + 1
        return self._codec_packed("decode_aperiodicity_packed", coded, f_offsets, "out", fs, fft_size, None, W, out)

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
                                aperiodicity_full, x_lengths=None, harvest_options=None, dio_options=None,
                                cheaptrick_options=None, d4c_options=None):
        """analyze_batch on this rank's shard with every finished slice broadcast into the FULL arrays of all ranks.
        harvest_options / dio_options: a list of one option per utterance of THIS rank's shard.
        cheaptrick_options / d4c_options: the same for the spectral options
        (world_b200_analyze_batch_allgather_spectral_options).  The shards' largest sizes may differ, so the row_stride
        is the last dimension of the full arrays, which every rank allocates alike; ValueError when both are None."""
        n, stride = x.shape
        xl, keep = _int_array(x_lengths, n)
        outs = (_ptr(time_axis_full), _ptr(f0_full), time_axis_full.shape[1],
                _ptr(spectrogram_full) if spectrogram_full is not None else None,
                _ptr(aperiodicity_full) if aperiodicity_full is not None else None)
        self._chain("analyze_batch_allgather", (_ptr(x), n, stride, xl, fs, C.byref(option)), n, harvest_options,
                    dio_options, outs, cheaptrick_options=cheaptrick_options, d4c_options=d4c_options, device=True,
                    rows=(spectrogram_full, aperiodicity_full))

    def analyze_host(self, x_host, fs, option: AnalysisOption, x_lengths=None, time_axis=None, f0=None,
                     spectrogram=None, aperiodicity=None, f0_stride=None, harvest_options=None, dio_options=None,
                     cheaptrick_options=None, d4c_options=None):
        """Whole chain on HOST arrays (numpy or pinned torch CPU tensors); outputs are written
        into the given host arrays (allocated with numpy when None).  harvest_options / dio_options: a list of
        one option per utterance of the chain's F0 method.  cheaptrick_options / d4c_options: as for analyze_batch
        (world_b200_analyze_host_spectral_options); whole padded rows come back, 0 past each utterance's
        fft_size // 2 + 1 values and past its frames."""
        import numpy as np
        n, stride = x_host.shape
        frame_period = _frame_period(option)
        lens = [stride] * n if x_lengths is None else [int(v) for v in x_lengths]
        fl = [self.frames(fs, v, frame_period) for v in lens]
        f0_stride = f0_stride or max(fl)
        bins = _full_bins(option, cheaptrick_options)
        if time_axis is None:
            time_axis = np.zeros((n, f0_stride))
        if f0 is None:
            f0 = np.zeros((n, f0_stride))
        if spectrogram is None:
            spectrogram = np.zeros((n, f0_stride, bins))
        if aperiodicity is None:
            aperiodicity = np.zeros((n, f0_stride, bins))
        xl, keep = _int_array(x_lengths, n)
        self._chain("analyze_host", (_ptr(x_host), n, stride, xl, fs, C.byref(option)), n, harvest_options,
                    dio_options, (_ptr(time_axis), _ptr(f0), f0_stride, _ptr(spectrogram), _ptr(aperiodicity)),
                    cheaptrick_options=cheaptrick_options, d4c_options=d4c_options, rows=(spectrogram, aperiodicity))
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
                           dio_options=None, cheaptrick_options=None, d4c_options=None):
        """Whole chain with device-side ingest (nbit 0 = float64 rows, 16 = int16 rows, ...) and codec;
        only the coded rows are downloaded.  harvest_options / dio_options: a list of one option per utterance of
        the chain's F0 method (not both).  cheaptrick_options / d4c_options: as for analyze_coded_batch."""
        import numpy as np
        n = x_host.shape[0]
        item = x_host.element_size() if hasattr(x_host, "element_size") else x_host.itemsize
        stride = x_host.shape[1] * item // (nbit // 8 if nbit else 8)
        frame_period = _frame_period(option)
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
        self._chain("analyze_coded_host", (_ptr(x_host), nbit, n, stride, xl, fs, C.byref(option)), n, harvest_options,
                    dio_options, (number_of_dimensions, _ptr(time_axis), _ptr(f0), f0_stride, _ptr(coded_sp),
                                  _ptr(coded_ap)), cheaptrick_options=cheaptrick_options, d4c_options=d4c_options)
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
        frame_period = _frame_period(option)
        return x.shape[0], x.shape[1] * item // width, frame_period

    def analyze_coded_batch(self, x, nbit, fs, option: AnalysisOption, number_of_dimensions, x_lengths=None,
                            time_axis=None, f0=None, coded_sp=None, coded_ap=None, harvest_options=None,
                            dio_options=None, cheaptrick_options=None, d4c_options=None):
        """Whole chain on DEVICE arrays with coded rows out: analyze_batch's two internal streams, analyze_coded_host's
        formats.  x: float64 rows (nbit 0) or PCM rows (nbit 16: int16; 8/24/32: uint8 rows of nbit/8 bytes per
        sample); the PCM is converted slice by slice on the device.  Outputs are allocated on x's device when None
        and the work is enqueued on torch's current stream.  Returns (t, f0, coded_sp, coded_ap, frame counts) with
        coded_sp [n, L, number_of_dimensions] and coded_ap [n, L, max(1, GetNumberOfAperiodicities(fs))] (left zero
        below 12 kHz).  harvest_options / dio_options: a list of one option per utterance of the chain's F0 method.
        cheaptrick_options / d4c_options: a list of one CheapTrickOption / D4COption per utterance (D4C runs at each
        utterance's CheapTrick fft_size)."""
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
        self._chain("analyze_coded_batch", (_ptr(x), nbit, n, stride, xl, fs, C.byref(option)), n, harvest_options,
                    dio_options, (number_of_dimensions, _ptr(time_axis), _ptr(f0), time_axis.shape[1], _ptr(coded_sp),
                                  _ptr(coded_ap)), cheaptrick_options=cheaptrick_options, d4c_options=d4c_options,
                    device=True)
        return time_axis, f0, coded_sp, coded_ap, fl

    # -- voice transformation: analysis, modification and synthesis in one call --------------------------------
    def transform_samples(self, fs, x_length, frame_period=5.0, time_scale=1.0) -> int:
        """Output length of one utterance of transform(): the demo's y_length with frame period frame_period * time_scale
        (world_b200_transform_samples)."""
        return int(self.lib.world_b200_transform_samples(fs, x_length, frame_period, time_scale))

    def _transform_args(self, x, nbit, fs, option, f0_scale, spectral_ratio, time_scale, x_lengths, harvest_options,
                        dio_options, dtype, cheaptrick_options=None, d4c_options=None):
        """(n, y_stride, nbit_out, args, suffix): args run from nbit to nbit_out; suffix "_spectral_options" when
        cheaptrick_options or d4c_options is given (their arrays then follow the F0 option arrays)."""
        n, stride, frame_period = self._coded_rows(x, nbit, option)
        lens = [stride] * n if x_lengths is None else [int(v) for v in x_lengths]
        ts = _factors(time_scale, n, "time_scale")
        y_lens = [self.transform_samples(fs, v, frame_period, ts[u] if ts is not None else 1.0)
                  for u, v in enumerate(lens)]
        xl, _ = _int_array(x_lengths, n)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        nbit_out = 16 if _pcm16(dtype) else 0
        y_stride = max(y_lens + [1])
        spectral = []
        if cheaptrick_options is not None or d4c_options is not None:
            spectral = [None if cheaptrick_options is None else _option_array(CheapTrickOption, cheaptrick_options, n),
                        None if d4c_options is None else _option_array(D4COption, d4c_options, n)]
        args = [nbit, n, stride, xl, fs, C.byref(option), per_utt, per_dio, *spectral,
                _factors(f0_scale, n, "f0_scale"), _factors(spectral_ratio, n, "spectral_ratio"), ts, nbit_out]
        return n, y_stride, nbit_out, args, "_spectral_options" if spectral else ""

    def transform(self, x, nbit, fs, option: AnalysisOption, f0_scale=None, spectral_ratio=None, time_scale=None,
                  x_lengths=None, harvest_options=None, dio_options=None, dtype=None, cheaptrick_options=None,
                  d4c_options=None):
        """The reference demo's loop on DEVICE arrays in one call (world_b200_transform_batch): analysis with option's F0
        method, CheapTrick and D4C, f0 scaled by f0_scale and the envelope stretched by spectral_ratio (as modify()),
        and Synthesis with the frame period scaled by time_scale (above 1: slower).  Each factor may be None, one number,
        or one value per utterance.  x as for analyze_coded_batch (float64 rows for nbit 0, else PCM rows).  Returns
        (y, y_lengths): y [n, max y_length] float64, or int16 for dtype int16 (wavwrite's quantisation), on x's device,
        with samples past an utterance's length left 0; y_lengths from transform_samples.  Every row equals
        analyze_batch -> modify -> synthesis of the same utterance bit for bit.  cheaptrick_options / d4c_options: a
        list of one option per utterance (world_b200_transform_batch_spectral_options): utterance u is analysed,
        modified and synthesised at cheaptrick_options[u].fft_size."""
        n, y_stride, nbit_out, args, suffix = self._transform_args(x, nbit, fs, option, f0_scale, spectral_ratio,
                                                                   time_scale, x_lengths, harvest_options, dio_options,
                                                                   dtype, cheaptrick_options, d4c_options)
        if self.xp == "torch":
            y = self.torch.zeros((n, y_stride), dtype=self.torch.int16 if nbit_out else self.torch.float64,
                                 device=x.device)
        else:
            import numpy as np
            y = np.zeros((n, y_stride), dtype=np.int16 if nbit_out else np.float64)
        yl = (C.c_int * max(n, 1))()
        self._use_current_stream()
        self._check(getattr(self.lib, f"world_b200_transform_batch{suffix}")(self._h, _ptr(x), *args, _ptr(y),
                                                                              y_stride, yl))
        return y, list(yl)[:n]

    def transform_host(self, x, nbit, fs, option: AnalysisOption, f0_scale=None, spectral_ratio=None, time_scale=None,
                       x_lengths=None, harvest_options=None, dio_options=None, dtype=None, out=None,
                       cheaptrick_options=None, d4c_options=None):
        """transform() for HOST arrays (numpy or CPU tensors; world_b200_transform_host): PCM chunks are uploaded,
        transformed and downloaded pipelined, so only PCM crosses PCIe.  Returns (y, y_lengths) with y a host array of
        whole rows (0 past each length).  out: a contiguous [n, max y_length] host array of the output dtype to write
        into (a pinned one lets the copies overlap the kernels).  cheaptrick_options / d4c_options as in transform()."""
        import numpy as np
        n, y_stride, nbit_out, args, suffix = self._transform_args(x, nbit, fs, option, f0_scale, spectral_ratio,
                                                                   time_scale, x_lengths, harvest_options, dio_options,
                                                                   dtype, cheaptrick_options, d4c_options)
        want = np.int16 if nbit_out else np.float64
        if out is None:
            out = np.zeros((n, y_stride), dtype=want)
        y = out.numpy() if hasattr(out, "numpy") else out
        if y.shape != (n, y_stride) or y.dtype != want or not y.flags.c_contiguous:
            raise ValueError(f"out: a contiguous [{n}, {y_stride}] {np.dtype(want).name} host array")
        xh = x.numpy() if hasattr(x, "numpy") else x
        if not xh.flags.c_contiguous:
            raise ValueError("x: a contiguous host array")
        yl = (C.c_int * max(n, 1))()
        self._check(getattr(self.lib, f"world_b200_transform_host{suffix}")(self._h, _ptr(xh), *args, _ptr(y),
                                                                             y_stride, yl))
        return out, list(yl)[:n]

    # -- the voice transformation on packed batches: utterance u = samples [x_offsets[u], x_offsets[u + 1]) in and
    #    samples [y_offsets[u], y_offsets[u + 1]) out ------------------------------------------------------------------
    def transform_packed_samples(self, fs, x_offsets, frame_period=5.0, time_scale=None):
        """The output offsets of a packed transform (numpy int64, n + 1; world_b200_transform_packed_samples): utterance
        u's output is samples [y[u], y[u + 1]), of transform_samples(fs, its length, frame_period, time_scale[u])."""
        import numpy as np
        n, xo = _offsets(x_offsets)
        y = (C.c_longlong * (n + 1))()
        rc = self.lib.world_b200_transform_packed_samples(fs, n, xo, frame_period, _factors(time_scale, n, "time_scale"),
                                                          y)
        if rc:
            raise WorldError(f"world_b200_transform_packed_samples: bad x_offsets, time_scale or arguments (code {rc})")
        return np.array(y[:], dtype=np.int64)

    def _transform_packed(self, name, x, nbit, x_offsets, fs, option, f0_scale, spectral_ratio, time_scale,
                          harvest_options, dio_options, cheaptrick_options, d4c_options, dtype, y, host, curves=None):
        """Calls world_b200_<name> on a packed batch: (y [Y], y_offsets as numpy int64), y allocated when None (device:
        on x's device; host: numpy)."""
        import numpy as np
        n, xo = _offsets(x_offsets)
        per_utt, per_dio = _chain_options(harvest_options, dio_options, n)
        ct = None if cheaptrick_options is None else _option_array(CheapTrickOption, cheaptrick_options, n)
        d4 = None if d4c_options is None else _option_array(D4COption, d4c_options, n)
        pcm16 = _pcm16(dtype)
        try:
            Y = int(self.transform_packed_samples(fs, x_offsets, _frame_period(option), time_scale)[-1])
        except WorldError:   # the call below names what is wrong
            Y = 0
        if host:
            want = np.int16 if pcm16 else np.float64
            if y is None:
                y = np.empty((Y,), dtype=want)
            yh = y.numpy() if hasattr(y, "numpy") else y
            if yh.shape != (Y,) or yh.dtype != want or not yh.flags.c_contiguous:
                raise ValueError(f"out: a contiguous [{Y}] {np.dtype(want).name} host array")
            xh = x.numpy() if hasattr(x, "numpy") else x
            if not xh.flags.c_contiguous:
                raise ValueError("x: a contiguous host array")
            xp, yp = _ptr(xh), _ptr(yh)
        else:
            if y is None:
                y = self._packed_y(x, Y, pcm16)
            xp, yp = _ptr(x), _ptr(y)
            self._use_current_stream()
        got = (C.c_longlong * (n + 1))()
        if curves is None:
            pitch, formant = _factors(f0_scale, n, "f0_scale"), _factors(spectral_ratio, n, "spectral_ratio")
        else:
            pitch, formant = curves
        self._check(getattr(self.lib, f"world_b200_{name}")(
            self._h, xp, nbit, n, xo, fs, C.byref(option), per_utt, per_dio, ct, d4, pitch, formant,
            _factors(time_scale, n, "time_scale"), 16 if pcm16 else 0, yp, got))
        return y, np.array(got[:], dtype=np.int64)

    def transform_packed(self, x, nbit, x_offsets, fs, option: AnalysisOption, f0_scale=None, spectral_ratio=None,
                         time_scale=None, harvest_options=None, dio_options=None, cheaptrick_options=None,
                         d4c_options=None, dtype=None, y=None):
        """transform() on a PACKED batch of DEVICE samples (world_b200_transform_packed): x holds float64 samples (nbit
        0) or nbit-bit PCM back to back, utterance u being samples [x_offsets[u], x_offsets[u + 1]) (x_offsets: n + 1
        offsets, a list, numpy array or CPU tensor).  Returns (y [Y], y_offsets [n + 1]) on x's device: float64, or
        int16 for dtype int16; utterance u's output is samples [y_offsets[u], y_offsets[u + 1]).  Each utterance's
        samples equal transform()'s row of the same utterance padded, bit for bit.  Factors and option lists as in
        transform(); y: a [Y] device array to write into."""
        return self._transform_packed("transform_packed", x, nbit, x_offsets, fs, option, f0_scale, spectral_ratio,
                                      time_scale, harvest_options, dio_options, cheaptrick_options, d4c_options, dtype,
                                      y, host=False)

    def transform_host_packed(self, x, nbit, x_offsets, fs, option: AnalysisOption, f0_scale=None,
                              spectral_ratio=None, time_scale=None, harvest_options=None, dio_options=None,
                              cheaptrick_options=None, d4c_options=None, dtype=None, out=None):
        """transform_packed for HOST arrays (numpy or CPU tensors; world_b200_transform_host_packed): chunks of
        utterances go up and come back as one copy each.  Returns (y [Y], y_offsets) with y a host array.  out: a
        contiguous [Y] host array of the output dtype to write into (a pinned one lets the copies overlap the
        kernels)."""
        return self._transform_packed("transform_host_packed", x, nbit, x_offsets, fs, option, f0_scale,
                                      spectral_ratio, time_scale, harvest_options, dio_options, cheaptrick_options,
                                      d4c_options, dtype, out, host=True)

    def transform_packed_curves(self, x, nbit, x_offsets, fs, option: AnalysisOption, f0_curve=None,
                                spectral_ratio_curve=None, time_scale=None, harvest_options=None, dio_options=None,
                                cheaptrick_options=None, d4c_options=None, dtype=None, y=None):
        """transform_packed with pitch and formant curves (world_b200_transform_packed_curves): f0_curve and
        spectral_ratio_curve are [F] DEVICE arrays of one factor per analysis frame, at the frame offsets
        packed_frames(fs, x_offsets, frame_period) gives (either may be None); time_scale stays one per utterance.
        Every utterance's output equals analyze_packed -> modify_curves_packed -> synthesis_packed at
        frame_period * time_scale[u], bit for bit.  Returns (y [Y], y_offsets) as transform_packed."""
        return self._transform_packed("transform_packed_curves", x, nbit, x_offsets, fs, option, None, None,
                                      time_scale, harvest_options, dio_options, cheaptrick_options, d4c_options, dtype,
                                      y, host=False, curves=(_curve(f0_curve), _curve(spectral_ratio_curve)))

    def transform_host_packed_curves(self, x, nbit, x_offsets, fs, option: AnalysisOption, f0_curve=None,
                                     spectral_ratio_curve=None, time_scale=None, harvest_options=None,
                                     dio_options=None, cheaptrick_options=None, d4c_options=None, dtype=None,
                                     out=None):
        """transform_packed_curves for HOST arrays (world_b200_transform_host_packed_curves): x, out and the [F]
        curves are host arrays (numpy or CPU tensors); each chunk's curve frames go up beside its samples.  Returns
        (y [Y], y_offsets) as transform_host_packed."""
        import numpy as np
        keep = [None if c is None else np.ascontiguousarray(c.numpy() if hasattr(c, "numpy") else c,
                                                            dtype=np.float64) for c in (f0_curve, spectral_ratio_curve)]
        return self._transform_packed("transform_host_packed_curves", x, nbit, x_offsets, fs, option, None, None,
                                      time_scale, harvest_options, dio_options, cheaptrick_options, d4c_options, dtype,
                                      out, host=True, curves=tuple(_ptr(c) for c in keep))

    def analyze_coded_batch_allgather(self, x, nbit, fs, option: AnalysisOption, number_of_dimensions, time_axis_full,
                                      f0_full, coded_sp_full, coded_ap_full, x_lengths=None, harvest_options=None,
                                      dio_options=None, cheaptrick_options=None, d4c_options=None):
        """analyze_coded_batch on this rank's shard with every finished slice sent into the FULL arrays of all ranks
        (the coded rows are what crosses between GPUs).  coded_sp_full / coded_ap_full may be None to skip CheapTrick /
        D4C.  harvest_options / dio_options / cheaptrick_options / d4c_options: a list of one option per utterance of
        THIS rank's shard (world_b200_analyze_coded_batch_allgather_spectral_options for the spectral ones)."""
        n, stride, _ = self._coded_rows(x, nbit, option)
        xl, keep = _int_array(x_lengths, n)
        self._chain("analyze_coded_batch_allgather", (_ptr(x), nbit, n, stride, xl, fs, C.byref(option)), n,
                    harvest_options, dio_options, (number_of_dimensions, _ptr(time_axis_full), _ptr(f0_full),
                                                   time_axis_full.shape[1], _ptr(coded_sp_full), _ptr(coded_ap_full)),
                    cheaptrick_options=cheaptrick_options, d4c_options=d4c_options, device=True)
