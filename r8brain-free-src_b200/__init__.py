"""r8brain-free-src_b200 -- Python mirror of the reference's resampler interface over the H100 C-ABI.

The product is libr8bgpu.so (hand-written sm_90a kernels + host planner, see csrc/ and
include/r8bgpu.h).  This module is a thin ctypes binding that mirrors the reference's
front-end names and argument meaning for the process() path:

    r8b::CDSPResampler(Src, Dst, MaxInLen, ReqTransBand=2, ReqAtten=206.91)   CDSPResampler.h:117-120
    r8b::CDSPResampler16 / 16IR / 24                                           CDSPResampler.h:729-810
    process / clear / oneshot / getMaxOutLen / getInLenBeforeOutPos /
    getInputRequiredForOutput / getInLenBeforeOutStart / getLatency[Frac]      CDSPResampler.h:406-651

plus `ResamplerBatch`, the channel-batched form of example.cpp:30-67 (one resampler per channel,
same block length for every channel).  There is no CPU fallback: constructing a batch without a
CUDA device raises.  The directory name contains '-', so import it through
`__graft_entry__.load_package()` (registers it as module `r8brain_free_src_b200`).
"""
import ctypes as C
import os
from fractions import Fraction

import numpy as np

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None

STAGE_NAMES = {0: "blockconv", 1: "frac_whole", 2: "frac_poly", 3: "hbup", 4: "hbdown"}
ATTEN_16 = 136.45   # CDSPResampler16   (CDSPResampler.h:745-746)
ATTEN_16IR = 109.56  # CDSPResampler16IR (:776-777)
ATTEN_24 = 180.15   # CDSPResampler24   (:806-807)


class StageInfo(C.Structure):
    _fields_ = [("kind", C.c_int), ("up", C.c_int), ("down", C.c_int), ("kernel_len", C.c_int),
                ("latency", C.c_int), ("ref_input_len", C.c_int), ("block_len_bits", C.c_int),
                ("fracs", C.c_int), ("in_step", C.c_int), ("out_step", C.c_int), ("order", C.c_int),
                ("max_out_len", C.c_int), ("atten", C.c_double), ("data_len", C.c_int)]


# r8bgpu_fused_info (include/r8bgpu.h): how a batch runs a BlockConvolver stage and the interpolator behind it
FUSED_NONE, FUSED_F2_TC, FUSED_F2_FMA, FUSED_V1_SMEM, FUSED_V1_GLOBAL, FUSED_F2_COPY, FUSED_ORDER2 = range(7)
FUSED_KERNELS = {FUSED_NONE: "none", FUSED_F2_TC: "f2-tc", FUSED_F2_FMA: "f2-fma", FUSED_V1_SMEM: "v1-smem",
                 FUSED_V1_GLOBAL: "v1-global", FUSED_F2_COPY: "f2-copy", FUSED_ORDER2: "order2"}


class FusedInfo(C.Structure):
    _fields_ = [("kernel", C.c_int), ("up", C.c_int), ("copy", C.c_int), ("in_step", C.c_int), ("out_step", C.c_int),
                ("tc_n_groups", C.c_int), ("tc_smaxp", C.c_int), ("ir", C.c_int), ("fma_n_groups", C.c_int),
                ("fma_smaxp", C.c_int), ("pad", C.c_int), ("ysh", C.c_int), ("tc_fits", C.c_int), ("fma_fits", C.c_int),
                ("cs", C.c_int), ("bank_in_smem", C.c_int)]


# r8bgpu_hb_info (include/r8bgpu.h): how a batch runs a half-band stage -- alone or in a cascade, and its tile plan
HB_SINGLE, HB_UP_CASCADE, HB_DOWN_CASCADE, HB_INSIDE = range(4)
HB_KINDS = {HB_SINGLE: "single", HB_UP_CASCADE: "up-cascade", HB_DOWN_CASCADE: "down-cascade", HB_INSIDE: "inside"}


class HbInfo(C.Structure):
    _fields_ = [("kind", C.c_int), ("first", C.c_int), ("n_stages", C.c_int), ("ntaps", C.c_int * 6),
                ("fuse_last2", C.c_int), ("n_buffers", C.c_int), ("w", C.c_int), ("smem_bytes", C.c_int),
                ("lo_off", C.c_int * 7), ("hi_off", C.c_int * 7), ("back", C.c_int * 7), ("writes_ring", C.c_int)]


# r8bgpu_blockconv_info (include/r8bgpu.h): the kernel and tile of a BlockConvolver stage
BC_FUSED, BC_F2_COPY, BC_BLOCKCONV, BC_LARGE = range(4)
BC_KERNELS = {BC_FUSED: "fused", BC_F2_COPY: "f2-copy", BC_BLOCKCONV: "k_blockconv", BC_LARGE: "k_bcl"}


class BlockConvInfo(C.Structure):
    _fields_ = [("kernel", C.c_int), ("fft_log2", C.c_int), ("up", C.c_int), ("src_up", C.c_int), ("down", C.c_int),
                ("block_exact", C.c_int), ("trunc", C.c_int), ("nyq_bin", C.c_int), ("lg", C.c_int), ("adv", C.c_int),
                ("smem_bytes", C.c_int), ("r0", C.c_int), ("scratch_tiles", C.c_int),
                ("scratch_bytes_per_ch", C.c_longlong), ("group_ch", C.c_int)]


# r8bgpu_frac_info (include/r8bgpu.h): the kernel and tiles of an interpolator stage
FRAC_FUSED, FRAC_WHOLE, FRAC_POLY = range(3)
FRAC_KERNELS = {FRAC_FUSED: "fused", FRAC_WHOLE: "k_frac<false>", FRAC_POLY: "k_frac<true>"}


class FracInfo(C.Structure):
    _fields_ = [("kernel", C.c_int), ("flen", C.c_int), ("fll", C.c_int), ("fracs", C.c_int), ("tile", C.c_int),
                ("window", C.c_int), ("tile_ragged", C.c_int), ("window_ragged", C.c_int), ("frac_cap", C.c_int)]



class Order2Info(C.Structure):
    _fields_ = [("poly_v2", C.c_int), ("n_tiles", C.c_int), ("span", C.c_int), ("span_max", C.c_int),
                ("poly_dir", C.c_int), ("poly_rows_cap", C.c_int), ("poly_row_stride", C.c_int), ("poly_chunks", C.c_int),
                ("poly_n", C.c_int), ("ysh", C.c_int), ("smem_bytes", C.c_int), ("flen", C.c_int), ("fracs", C.c_int),
                ("ratio", C.c_double)]

# Every symbol include/r8bgpu.h declares: name -> (restype, argtypes)
_SYMBOLS = {
    "r8bgpu_last_error": (C.c_char_p, []),
    "r8bgpu_version": (C.c_char_p, []),
    "r8bgpu_plan_create": (C.c_void_p, [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_int]),
    "r8bgpu_plan_create_stage": (C.c_void_p, [C.c_int, C.POINTER(C.c_double), C.c_int, C.c_int, C.c_int]),
    "r8bgpu_plan_destroy": (None, [C.c_void_p]),
    "r8bgpu_plan_max_out_len": (C.c_int, [C.c_void_p]),
    "r8bgpu_plan_in_len_before_out_pos": (C.c_int, [C.c_void_p, C.c_int]),
    "r8bgpu_plan_input_required_for_output": (C.c_int, [C.c_void_p, C.c_int]),
    "r8bgpu_plan_latency_frac": (C.c_double, [C.c_void_p]),
    "r8bgpu_plan_is_passthrough": (C.c_int, [C.c_void_p]),
    "r8bgpu_plan_stage_count": (C.c_int, [C.c_void_p]),
    "r8bgpu_plan_stage_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(StageInfo)]),
    "r8bgpu_plan_stage_data": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    "r8bgpu_plan_describe": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "r8bgpu_plan_simulate": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)]),
    "r8bgpu_plan_fused_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(FusedInfo)]),
    "r8bgpu_plan_cascade_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(HbInfo)]),
    "r8bgpu_plan_blockconv_info": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(BlockConvInfo)]),
    "r8bgpu_plan_frac_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(FracInfo)]),
    "r8bgpu_plan_order2_info": (C.c_int, [C.c_void_p, C.c_int, C.c_double, C.c_int, C.POINTER(Order2Info)]),
    "r8bgpu_device_count": (C.c_int, []),
    "r8bgpu_batch_create": (C.c_void_p, [C.c_void_p, C.c_int, C.c_int]),
    "r8bgpu_batch_destroy": (None, [C.c_void_p]),
    "r8bgpu_batch_shard_count": (C.c_int, [C.c_void_p]),
    "r8bgpu_batch_shard_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "r8bgpu_batch_shard": (C.c_void_p, [C.c_void_p, C.c_int]),
    "r8bgpu_batch_host_alloc": (C.c_void_p, [C.c_void_p, C.c_size_t, C.c_int]),
    "r8bgpu_batch_clear": (C.c_int, [C.c_void_p]),
    "r8bgpu_batch_channels": (C.c_int, [C.c_void_p]),
    "r8bgpu_batch_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_process": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.c_int]),
    "r8bgpu_batch_process_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.c_int]),
    "r8bgpu_batch_process_fmt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    "r8bgpu_batch_process_host_fmt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    "r8bgpu_batch_sync": (C.c_int, [C.c_void_p]),
    "r8bgpu_plan_simulate_ragged": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_process_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "r8bgpu_batch_process_host_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "r8bgpu_batch_process_ragged_fmt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "r8bgpu_batch_process_host_ragged_fmt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "r8bgpu_batch_clear_channels": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "r8bgpu_batch_channel_groups": (C.c_int, [C.c_void_p]),
    "r8bgpu_batch_flush": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "r8bgpu_batch_flush_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "r8bgpu_batch_channel_totals": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "r8bgpu_plan_flush_max_out_len": (C.c_int, [C.c_void_p]),
    "r8bgpu_plan_simulate_flush": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong),
                                             C.POINTER(C.c_int)]),
    "r8bgpu_batch_create_mixed": (C.c_void_p, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]),
    "r8bgpu_batch_max_out_len": (C.c_int, [C.c_void_p]),
    "r8bgpu_batch_flush_max_out_len": (C.c_int, [C.c_void_p]),
    "r8bgpu_batch_part": (C.c_void_p, [C.c_void_p, C.c_int]),
    "r8bgpu_plan_create_trim": (C.c_void_p, [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, C.c_double]),
    "r8bgpu_plan_create_asrc": (C.c_void_p, [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, C.c_double]),
    "r8bgpu_plan_max_trim": (C.c_double, [C.c_void_p]),
    "r8bgpu_plan_simulate_trim": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]),
    "r8bgpu_batch_set_trim": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "r8bgpu_batch_trim": (C.c_int, [C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_set_dither": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "r8bgpu_dither_quantize_host": (C.c_int, [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int, C.c_longlong, C.c_void_p,
                                              C.c_void_p]),
    "r8bgpu_batch_set_dsd_out": (C.c_int, [C.c_void_p, C.c_int]),
    "r8bgpu_batch_dsd_overloads": (C.c_int, [C.c_void_p, C.c_void_p]),
    "r8bgpu_dsd_modulate_host": (C.c_int, [C.c_double, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r8bgpu_plan_state_bytes": (C.c_size_t, [C.c_void_p]),
    "r8bgpu_plan_state_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "r8bgpu_plan_state_fingerprint": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "r8bgpu_batch_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "r8bgpu_batch_import": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "r8bgpu_batch_export_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "r8bgpu_batch_import_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "r8bgpu_plan_oneshot_warmup": (C.c_longlong, [C.c_void_p]),
    "r8bgpu_plan_simulate_oneshot": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_int]),
    "r8bgpu_batch_oneshot": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_oneshot_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_oneshot_adjoint": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_oneshot_mixed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p]),
    "r8bgpu_batch_oneshot_mixed_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_oneshot_adjoint_mixed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_void_p]),
    "r8bgpu_plan_oneshot_adjoint_extents": (C.c_longlong, [C.c_void_p, C.c_longlong, C.c_longlong, C.c_void_p, C.c_int]),
    "r8bgpu_plan_oneshot_adjoint_bytes": (C.c_longlong, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_oneshot_crops": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_oneshot_crops_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    "r8bgpu_batch_oneshot_crops_adjoint": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_int, C.c_void_p, C.c_void_p]),
    "r8bgpu_plan_simulate_oneshot_crops": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                     C.c_void_p, C.c_void_p, C.c_int]),
    "r8bgpu_plan_oneshot_crop_extents": (C.c_longlong, [C.c_void_p, C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong,
                                                        C.c_void_p, C.c_void_p, C.c_int]),
    "r8bgpu_batch_kernel_launches": (C.c_ulonglong, [C.c_void_p]),
    "r8bgpu_batch_device_bytes": (C.c_ulonglong, [C.c_void_p]),
    "r8bgpu_batch_stage_kernel": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, C.c_int]),
    "r8bgpu_batch_last_variant": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, C.c_int]),
    "r8bgpu_batch_set_timing": (C.c_int, [C.c_void_p, C.c_int]),
    "r8bgpu_batch_stage_time_ms": (C.c_double, [C.c_void_p, C.c_int, C.POINTER(C.c_ulonglong)]),
    "r8bgpu_measure_fp64_tflops": (C.c_double, [C.c_int]),
    "r8bgpu_host_alloc": (C.c_void_p, [C.c_size_t]),
    "r8bgpu_host_free": (None, [C.c_void_p]),
}


class R8bGpuError(RuntimeError):
    pass


# r8bgpu_sample_format / r8bgpu_buffer (include/r8bgpu.h)
# U8: unsigned 8-bit PCM; ULAW / ALAW: G.711 mu-law / A-law bytes (uint8 arrays, passed with fmt= / out_fmt=)
# DSD_LSB / DSD_MSB: one-bit DSD (DSF / DSDIFF bit order), uint8 arrays of bytes holding 8 samples each, with fmt=; as
# out_fmt= on a batch with DSD output on (Batch.set_dsd_out)
F64, F32, S16, S24, S32, U8, ULAW, ALAW = 0, 1, 2, 3, 4, 5, 6, 7
DSD_LSB, DSD_MSB = 16, 17
FORMAT_BYTES = {F64: 8, F32: 4, S16: 2, S24: 3, S32: 4, U8: 1, ULAW: 1, ALAW: 1, DSD_LSB: 1, DSD_MSB: 1}  # per element
# samples per element (buffer widths count elements, lengths count samples)
FORMAT_SAMPLES = {DSD_LSB: 8, DSD_MSB: 8}
_NP_FORMATS = {"float64": F64, "float32": F32, "int16": S16, "int32": S32, "uint8": U8}
# the numpy element type of each format's buffers (S24: uint8 [..., 3])
_NP_DTYPES = {F64: np.float64, F32: np.float32, S16: np.int16, S32: np.int32, S24: np.uint8, U8: np.uint8, ULAW: np.uint8,
              ALAW: np.uint8, DSD_LSB: np.uint8, DSD_MSB: np.uint8}


def _default_out(fi):
    """The output format when none is given: the input's, or float64 for the input-only DSD formats."""
    return F64 if fi in (DSD_LSB, DSD_MSB) else fi


def _dtype_format(dt):
    """Sample format of a numpy or torch dtype."""
    return _NP_FORMATS[np.dtype(str(dt).replace("torch.", "")).name]


# r8bgpu_dither (include/r8bgpu.h, "dithered integer output")
DITHER_OFF, DITHER_TPDF, DITHER_MAX_TAPS = 0, 1, 16


class Dither(C.Structure):
    _fields_ = [("kind", C.c_int), ("seed", C.c_ulonglong), ("n_taps", C.c_int), ("taps", C.c_double * DITHER_MAX_TAPS)]

    @classmethod
    def make(cls, seed, taps=None, kind=DITHER_TPDF):
        t = [] if taps is None else [float(v) for v in np.asarray(taps, dtype=np.float64).reshape(-1)]
        d = cls(int(kind), int(seed) & 0xFFFFFFFFFFFFFFFF, len(t))
        for k, v in enumerate(t[:DITHER_MAX_TAPS]):
            d.taps[k] = v
        if len(t) > DITHER_MAX_TAPS:
            d.n_taps = len(t)  # refused by the library with its message
        return d


def dither_quantize(y, fmt, seed, taps=None, scale=1.0, first_index=0, state=None, kind=DITHER_TPDF):
    """The dithered quantiser on the host (r8bgpu_dither_quantize_host), bit for bit what a batch set with
    Batch.set_dither(.., seed, taps) stores for outputs first_index .. of one channel whose fp64 outputs are y.
    fmt: S16, S24, S32, U8, ULAW or ALAW.  state: the error history (16 float64, newest first, zeros after a clear), updated in
    place; pass the same array to continue a stream.  Returns (q, state): int16 / int32, packed uint8 [n, 3] for S24, or uint8
    for U8, ULAW and ALAW."""
    y = np.ascontiguousarray(y, dtype=np.float64).reshape(-1)
    if state is None:
        state = np.zeros(DITHER_MAX_TAPS, dtype=np.float64)
    if state.dtype != np.float64 or state.shape != (DITHER_MAX_TAPS,) or not state.flags.c_contiguous:
        raise ValueError("state must be a contiguous float64 array of 16")
    q = {S16: lambda: np.zeros(len(y), np.int16), S32: lambda: np.zeros(len(y), np.int32),
         S24: lambda: np.zeros((len(y), 3), np.uint8), U8: lambda: np.zeros(len(y), np.uint8),
         ULAW: lambda: np.zeros(len(y), np.uint8), ALAW: lambda: np.zeros(len(y), np.uint8)}.get(
        fmt, lambda: np.zeros(max(len(y), 1), np.int32))()
    d = Dither.make(seed, taps, kind)
    if lib().r8bgpu_dither_quantize_host(C.byref(d), int(fmt), float(scale), y.ctypes.data, len(y), int(first_index),
                                         state.ctypes.data, q.ctypes.data) != 0:
        raise R8bGpuError(_err())
    return q, state


def dsd_modulate(y, scale=1.0, state=None):
    """The one-bit DSD modulator on the host (r8bgpu_dsd_modulate_host), bit for bit what a batch with DSD output on
    writes for one channel whose fp64 outputs are y.  state: 8 float64 (zeros after a clear), updated in place.
    Returns (bits, overloads): uint8 0 / 1 per sample (np.packbits(bits, bitorder="little") gives DSF bytes)."""
    y = np.ascontiguousarray(y, dtype=np.float64)
    st = np.zeros(8) if state is None else state
    if st.dtype != np.float64 or st.shape != (8,) or not st.flags.c_contiguous:
        raise ValueError("state must be a contiguous float64 array of 8")
    bits = np.zeros(len(y), dtype=np.uint8)
    ov = C.c_longlong(0)
    if lib().r8bgpu_dsd_modulate_host(float(scale), y.ctypes.data, len(y), st.ctypes.data, bits.ctypes.data,
                                      C.byref(ov)) != 0:
        raise R8bGpuError(_err())
    return bits, ov.value


# r8bgpu_oneshot_seg (include/r8bgpu.h, "long clips")
ONESHOT_SEG = np.dtype([("clip", np.int32), ("lane", np.int32), ("round", np.int32), ("pad_", np.int32), ("start", np.int64),
                        ("p0", np.int64), ("p1", np.int64), ("e0", np.int64), ("e1", np.int64)])

# r8bgpu_crop (include/r8bgpu.h, "crops of long clips")
CROP = np.dtype([("clip", np.int32), ("pad_", np.int32), ("o0", np.int64), ("o1", np.int64)])


def _crops(crops):
    """crops ([n, 3] of (clip, o0, o1)) as a contiguous r8bgpu_crop array."""
    c = np.asarray(crops, dtype=np.int64).reshape(-1, 3)
    out = np.zeros(len(c), dtype=CROP)
    out["clip"], out["o0"], out["o1"] = c[:, 0], c[:, 1], c[:, 2]
    return out


def _clip_dither(dither, n_clips):
    """dither (None, or per clip: a seed, a Dither or None for off) as an r8bgpu_dither array of n_clips."""
    if dither is None:
        return None
    dv = (Dither * max(n_clips, 1))()
    for r, sd in enumerate(dither):
        if isinstance(sd, Dither):
            dv[r] = sd
        elif sd is not None:
            dv[r] = Dither.make(sd)
    return dv


def _rows_out(fi, out_fmt, dev, interleaved, n_rows, W, out_scale):
    """(y, bo): zeros of n_rows rows of W samples (interleaved: transposed) in out_fmt (default: _default_out(fi)), a host
    array (dev None) or a tensor on dev, and its buffer."""
    out_fmt = _default_out(fi) if out_fmt is None else out_fmt
    shape = ((W, n_rows) if interleaved else (n_rows, W)) + ((3,) if out_fmt == S24 else ())
    if dev is None:
        y = np.zeros(shape, dtype=_NP_DTYPES[out_fmt])
        yp = y.ctypes.data
    else:
        import torch
        y = torch.zeros(shape, dtype=getattr(torch, np.dtype(_NP_DTYPES[out_fmt]).name), device=dev)
        yp = y.data_ptr()
    return y, Buffer.make(yp, out_fmt, interleaved, max(n_rows, 1) if interleaved else W, out_scale)


def _grad_in(name, gy, interleaved):
    """An output gradient of the adjoints checked (name: the method, for messages): (gy contiguous, its rows, its width)."""
    import torch
    if not isinstance(gy, torch.Tensor) or not gy.is_cuda:
        raise TypeError(name + " takes a CUDA tensor")
    if gy.dtype not in (torch.float64, torch.float32):
        raise TypeError(name + " takes float64 or float32 gradients")
    gy = gy.contiguous()
    return (gy, gy.shape[1], gy.shape[0]) if interleaved else (gy, gy.shape[0], gy.shape[1])


def _elems(fmt, n):
    """Elements of format fmt holding n samples (DSD: bytes of 8)."""
    return n // FORMAT_SAMPLES.get(fmt, 1)


class Buffer(C.Structure):
    _fields_ = [("data", C.c_void_p), ("format", C.c_int), ("interleaved", C.c_int),
                ("stride", C.c_size_t), ("scale", C.c_double)]

    @classmethod
    def make(cls, ptr, fmt, interleaved, stride, scale=1.0):
        return cls(C.c_void_p(int(ptr) if ptr else None), int(fmt), int(bool(interleaved)), int(stride), float(scale))


def lib_path():
    return _build.LIB


def lib():
    """Load (building first if stale and nvcc is present) the C-ABI library."""
    global _lib
    if _lib is None:
        path = _build.build()
        L = C.CDLL(path)
        for name, (res, args) in _SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError here == header/library mismatch: fail loudly
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def _err():
    return lib().r8bgpu_last_error().decode("utf-8", "replace")


def device_count():
    return lib().r8bgpu_device_count()


def measure_fp64_tflops(device=-1):
    """Measured DFMA ceiling of the device (bench.py's secondary roofline)."""
    v = lib().r8bgpu_measure_fp64_tflops(int(device))
    if v < 0:
        raise R8bGpuError(_err())
    return v


class Plan:
    """Immutable stage chain + filters for (src, dst): what CDSPResampler's constructor decides."""

    def __init__(self, src_rate, dst_rate, max_in_len, trans_band=2.0, atten=206.91, phase=0,
                 extfft=0, fasttiming=0, _handle=None):
        self._h = _handle if _handle is not None else lib().r8bgpu_plan_create(
            float(src_rate), float(dst_rate), int(max_in_len), float(trans_band), float(atten),
            int(phase), int(extfft), int(fasttiming))
        if not self._h:
            raise R8bGpuError(_err())
        self.src_rate, self.dst_rate, self.max_in_len = float(src_rate), float(dst_rate), int(max_in_len)

    @classmethod
    def trim(cls, src_rate, dst_rate, max_in_len, trans_band, atten, max_trim, extfft=0):
        """A trim plan (r8bgpu_plan_create_trim): the chain for (src, dst) with its interpolator always the order-2 bank,
        whose ratio each channel of a batch may trim by a factor f in [1 - max_trim, 1 + max_trim] (Batch.set_trim);
        0 < max_trim <= 0.01.  Buffer lengths (max_out_len) are those of the largest factor."""
        h = lib().r8bgpu_plan_create_trim(float(src_rate), float(dst_rate), int(max_in_len), float(trans_band),
                                          float(atten), int(extfft), float(max_trim))
        if not h:
            raise R8bGpuError(_err())
        return cls(src_rate, dst_rate, max_in_len, _handle=h)

    @classmethod
    def asrc(cls, src_rate, dst_rate, max_in_len, trans_band, atten, max_trim, extfft=0):
        """A trim plan for any rate pair (r8bgpu_plan_create_asrc), src == dst and integer ratios included: where
        Plan.trim accepts the pair, the same plan; elsewhere the chain the reference builds at a rate next to (src, dst),
        whose order-2 interpolator each channel trims as on any trim plan.  Never a passthrough plan."""
        h = lib().r8bgpu_plan_create_asrc(float(src_rate), float(dst_rate), int(max_in_len), float(trans_band),
                                          float(atten), int(extfft), float(max_trim))
        if not h:
            raise R8bGpuError(_err())
        return cls(src_rate, dst_rate, max_in_len, _handle=h)

    @property
    def max_trim(self):
        """0 for an ordinary plan."""
        return lib().r8bgpu_plan_max_trim(self._h)

    def simulate_trim(self, lens, factors, timing=False):
        """One channel of a trim plan on the host scheduler (CPU only): block i of lens[i] samples is fed after factor
        factors[i] has been set.  Returns the per-call counts, or with timing=True (counts, next_pos, next_frac): the
        interpolator's read position (integer index and fraction of its next output) after each call."""
        lens = np.ascontiguousarray(lens, dtype=np.int32).reshape(-1)
        fs = np.ascontiguousarray(factors, dtype=np.float64).reshape(-1)
        if len(fs) != len(lens):
            raise ValueError("expected one factor per call")
        counts = np.zeros(len(lens), dtype=np.int32)
        pos = np.zeros(len(lens), dtype=np.int64)
        frac = np.zeros(len(lens), dtype=np.float64)
        if lib().r8bgpu_plan_simulate_trim(self._h, len(lens), lens.ctypes.data, fs.ctypes.data, counts.ctypes.data,
                                           pos.ctypes.data, frac.ctypes.data) != 0:
            raise R8bGpuError(_err())
        return (counts, pos, frac) if timing else counts

    @classmethod
    def single_stage(cls, kind, params, max_in_len, extfft=0):
        arr = (C.c_double * len(params))(*[float(p) for p in params])
        h = lib().r8bgpu_plan_create_stage(int(kind), arr, len(params), int(max_in_len), int(extfft))
        if not h:
            raise R8bGpuError(_err())
        return cls(0.0, 0.0, max_in_len, _handle=h)

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.r8bgpu_plan_destroy(self._h)
            self._h = None

    @property
    def max_out_len(self):
        return lib().r8bgpu_plan_max_out_len(self._h)

    @property
    def passthrough(self):
        return bool(lib().r8bgpu_plan_is_passthrough(self._h))

    def in_len_before_out_pos(self, pos):
        return lib().r8bgpu_plan_in_len_before_out_pos(self._h, int(pos))

    def input_required_for_output(self, n):
        return lib().r8bgpu_plan_input_required_for_output(self._h, int(n))

    def latency_frac(self):
        return lib().r8bgpu_plan_latency_frac(self._h)

    def stages(self):
        out = []
        for i in range(lib().r8bgpu_plan_stage_count(self._h)):
            info = StageInfo()
            if lib().r8bgpu_plan_stage_info(self._h, i, C.byref(info)) != 0:
                raise R8bGpuError(_err())
            d = {f: getattr(info, f) for f, _ in StageInfo._fields_}
            d["name"] = STAGE_NAMES[info.kind]
            out.append(d)
        return out

    def fused_info(self, i):
        """How a batch created now (under the current R8BGPU_* settings) would run BlockConvolver stage i and the
        interpolator behind it (r8bgpu_plan_fused_info; CPU only): a dict of the r8bgpu_fused_info fields, with
        "kernel" named as in FUSED_KERNELS."""
        info = FusedInfo()
        if lib().r8bgpu_plan_fused_info(self._h, int(i), C.byref(info)) != 0:
            raise R8bGpuError(_err())
        d = {f: getattr(info, f) for f, _ in FusedInfo._fields_}
        d["kernel"] = FUSED_KERNELS[info.kernel]
        return d

    def cascade_info(self, i):
        """How a batch created now (under the current R8BGPU_* settings) would run half-band stage i on its lock-step
        calls (r8bgpu_plan_cascade_info; CPU only): a dict of the r8bgpu_hb_info fields, with "kind" named as in
        HB_KINDS and the arrays cut to the cascade's stages (ntaps) and streams (lo_off, hi_off, back)."""
        info = HbInfo()
        if lib().r8bgpu_plan_cascade_info(self._h, int(i), C.byref(info)) != 0:
            raise R8bGpuError(_err())
        n = info.n_stages
        d = {f: getattr(info, f) for f, _ in HbInfo._fields_}
        d["kind"] = HB_KINDS[info.kind]
        d["ntaps"] = tuple(info.ntaps[:n])
        for f in ("lo_off", "hi_off", "back"):
            d[f] = tuple(getattr(info, f)[:n + 1])
        return d

    def blockconv_info(self, i, n_channels=1):
        """How a batch of n_channels created now (under the current R8BGPU_* settings) would run BlockConvolver stage i
        on its lock-step calls (r8bgpu_plan_blockconv_info; CPU only): a dict of the r8bgpu_blockconv_info fields, with
        "kernel" named as in BC_KERNELS."""
        info = BlockConvInfo()
        if lib().r8bgpu_plan_blockconv_info(self._h, int(i), int(n_channels), C.byref(info)) != 0:
            raise R8bGpuError(_err())
        d = {f: getattr(info, f) for f, _ in BlockConvInfo._fields_}
        d["kernel"] = BC_KERNELS[info.kernel]
        return d

    def frac_info(self, i):
        """How a batch created now (under the current R8BGPU_* settings) would run interpolator stage i
        (r8bgpu_plan_frac_info; CPU only): a dict of the r8bgpu_frac_info fields, with "kernel" named as in
        FRAC_KERNELS."""
        info = FracInfo()
        if lib().r8bgpu_plan_frac_info(self._h, int(i), C.byref(info)) != 0:
            raise R8bGpuError(_err())
        d = {f: getattr(info, f) for f, _ in FracInfo._fields_}
        d["kernel"] = FRAC_KERNELS[info.kernel]
        return d

    def order2_info(self, i, factor=1.0, span=0):
        """How a lock-step call would run the fused pair of BlockConvolver stage i and the order-2 interpolator behind it
        (r8bgpu_plan_order2_info; CPU only), at trim factor `factor` (1 on an ordinary plan) over `span` positions of the
        stream between the two stages (0: a full tile pair): a dict of the r8bgpu_order2_info fields."""
        info = Order2Info()
        if lib().r8bgpu_plan_order2_info(self._h, int(i), float(factor), int(span), C.byref(info)) != 0:
            raise R8bGpuError(_err())
        return {f: getattr(info, f) for f, _ in Order2Info._fields_}

    def stage_data(self, i):
        n = lib().r8bgpu_plan_stage_data(self._h, int(i), None, 0)
        if n < 0:
            raise R8bGpuError(_err())
        a = np.empty(n, dtype=np.float64)
        lib().r8bgpu_plan_stage_data(self._h, int(i), a.ctypes.data, n)
        return a

    def describe(self):
        n = lib().r8bgpu_plan_describe(self._h, None, 0)
        buf = C.create_string_buffer(n + 1)
        lib().r8bgpu_plan_describe(self._h, buf, n + 1)
        return buf.value.decode()

    def simulate(self, lens):
        """Per-call output counts the scheduler would return (CPU only, no GPU needed)."""
        lens = [int(v) for v in lens]
        a = (C.c_int * len(lens))(*lens)
        o = (C.c_int * len(lens))()
        if lib().r8bgpu_plan_simulate(self._h, a, len(lens), o) != 0:
            raise R8bGpuError(_err())
        return list(o)

    def simulate_ragged(self, lens, clear=None):
        """Per-channel counts of ragged calls on a batch (CPU only): lens [n_calls, n_channels]; clear (same shape,
        optional) names the channels cleared on their own just before each call.  Returns (counts [n_calls,
        n_channels], distinct channel schedules after each call)."""
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        n_calls, n_ch = lens.shape
        cl = None if clear is None else np.ascontiguousarray(clear, dtype=np.int32)
        if cl is not None and cl.shape != lens.shape:
            raise ValueError("clear must have the shape of lens")
        counts = np.empty_like(lens)
        groups = np.empty(n_calls, dtype=np.int32)
        if lib().r8bgpu_plan_simulate_ragged(self._h, n_ch, n_calls, lens.ctypes.data,
                                             None if cl is None else cl.ctypes.data, counts.ctypes.data,
                                             groups.ctypes.data) != 0:
            raise R8bGpuError(_err())
        return counts, groups

    @property
    def state_bytes(self):
        """Size of one channel's state blob (Batch.export_channels / import_channels); no GPU needed."""
        return int(lib().r8bgpu_plan_state_bytes(self._h))

    @property
    def state_fingerprint(self):
        """The plan's fingerprint as a state blob stores it (64 bytes): equal for equal plans."""
        buf = C.create_string_buffer(64)
        n = lib().r8bgpu_plan_state_fingerprint(self._h, buf, 64)
        return buf.raw[:n]

    def state_windows(self):
        """H_j per stage: the samples of stage input j a state blob carries (the plan's longest re-read reach)."""
        n = lib().r8bgpu_plan_state_windows(self._h, None, 0)
        w = np.zeros(max(n, 1), dtype=np.int64)
        lib().r8bgpu_plan_state_windows(self._h, w.ctypes.data, n)
        return w[:n]

    @property
    def flush_max_out_len(self):
        """Upper bound of what a default-target flush returns for any channel state (size flush buffers with it)."""
        return lib().r8bgpu_plan_flush_max_out_len(self._h)

    def default_target(self, n_in):
        """ceil(n_in * dst / src), exactly: the output length of a stream of n_in samples (the default flush target)."""
        q = Fraction(self.dst_rate) / Fraction(self.src_rate) * int(n_in)
        return -((-q.numerator) // q.denominator)

    @property
    def oneshot_warmup(self):
        """W: input samples each long-clip segment re-reads before its first kept output (a multiple of MaxInLen)."""
        return int(lib().r8bgpu_plan_oneshot_warmup(self._h))

    def simulate_oneshot(self, n_lanes, lens, oplens=None):
        """Dry run of Batch.oneshot_long on n_lanes lanes (r8bgpu_plan_simulate_oneshot, no GPU).  Returns (segs, n_calls):
        segs a structured array with fields clip, lane, round, start, p0, p1, e0, e1, by round and lane."""
        lens = np.ascontiguousarray(lens, dtype=np.int64).reshape(-1)
        op = None if oplens is None else np.ascontiguousarray(oplens, dtype=np.int64).reshape(-1)
        if op is not None and len(op) != len(lens):
            raise ValueError("expected one output length per clip")
        n_calls = C.c_int(0)
        args = (self._h, int(n_lanes), len(lens), lens.ctypes.data, None if op is None else op.ctypes.data, C.byref(n_calls))
        n = lib().r8bgpu_plan_simulate_oneshot(*args, None, 0)
        if n < 0:
            raise R8bGpuError(_err())
        segs = np.zeros(n, dtype=ONESHOT_SEG)
        if n and lib().r8bgpu_plan_simulate_oneshot(*args, segs.ctypes.data, n) != n:
            raise R8bGpuError(_err())
        return segs, int(n_calls.value)

    def simulate_oneshot_crops(self, n_lanes, lens, crops, oplens=None):
        """Dry run of Batch.oneshot_crops on n_lanes lanes (r8bgpu_plan_simulate_oneshot_crops, no GPU): crops [n, 3] of
        (clip, o0, o1).  Returns (segs, n_calls) as simulate_oneshot does; a segment's clip field is its CROP index."""
        lens = np.ascontiguousarray(lens, dtype=np.int64).reshape(-1)
        op = None if oplens is None else np.ascontiguousarray(oplens, dtype=np.int64).reshape(-1)
        if op is not None and len(op) != len(lens):
            raise ValueError("expected one output length per clip")
        cr = _crops(crops)
        n_calls = C.c_int(0)
        args = (self._h, int(n_lanes), len(lens), lens.ctypes.data, None if op is None else op.ctypes.data, len(cr),
                cr.ctypes.data if len(cr) else None, C.byref(n_calls))
        n = lib().r8bgpu_plan_simulate_oneshot_crops(*args, None, 0)
        if n < 0:
            raise R8bGpuError(_err())
        segs = np.zeros(n, dtype=ONESHOT_SEG)
        if n and lib().r8bgpu_plan_simulate_oneshot_crops(*args, segs.ctypes.data, n) != n:
            raise R8bGpuError(_err())
        return segs, int(n_calls.value)

    def oneshot_crop_extents(self, len, oplen, o0, o1):
        """(lo, hi) per stage (r8bgpu_plan_oneshot_crop_extents, no GPU): stage j's input samples [lo[j], hi[j]) are
        the ones outputs [o0, o1) of a clip of len samples with target oplen read.  Two int64 arrays."""
        args = (self._h, int(len), int(oplen), int(o0), int(o1))
        n = lib().r8bgpu_plan_oneshot_crop_extents(*args, None, None, 0)
        if n < 0:
            raise R8bGpuError(_err())
        lo, hi = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)
        if n and lib().r8bgpu_plan_oneshot_crop_extents(*args, lo.ctypes.data, hi.ctypes.data, int(n)) != n:
            raise R8bGpuError(_err())
        return lo, hi

    def oneshot_adjoint_extents(self, len, oplen):
        """R_j per stage (r8bgpu_plan_oneshot_adjoint_extents, no GPU): one past the largest index of stage j's input
        stream that an output in [0, oplen) of a clip of len samples reads.  An int64 array, one entry per stage."""
        n = lib().r8bgpu_plan_oneshot_adjoint_extents(self._h, int(len), int(oplen), None, 0)
        if n < 0:
            raise R8bGpuError(_err())
        ext = np.zeros(n, dtype=np.int64)
        if n and lib().r8bgpu_plan_oneshot_adjoint_extents(self._h, int(len), int(oplen), ext.ctypes.data, int(n)) != n:
            raise R8bGpuError(_err())
        return ext

    def oneshot_adjoint_bytes(self, lens, oplens=None):
        """Device scratch of Batch.oneshot_adjoint for these clips (r8bgpu_plan_oneshot_adjoint_bytes)."""
        lens = np.ascontiguousarray(lens, dtype=np.int64).reshape(-1)
        op = None if oplens is None else np.ascontiguousarray(oplens, dtype=np.int64).reshape(-1)
        n = lib().r8bgpu_plan_oneshot_adjoint_bytes(self._h, len(lens), lens.ctypes.data, None if op is None else op.ctypes.data)
        if n < 0:
            raise R8bGpuError(_err())
        return int(n)

    def simulate_flush(self, lens, target=None):
        """One stream fed blocks of lens[i] samples, then flushed to `target` (None: the default target), on the host
        scheduler (CPU only).  Returns (silence fed, samples the flush returns)."""
        lens = np.ascontiguousarray(lens, dtype=np.int32).reshape(-1)
        z, n = C.c_longlong(0), C.c_int(0)
        if lib().r8bgpu_plan_simulate_flush(self._h, len(lens), lens.ctypes.data, -1 if target is None else int(target),
                                            C.byref(z), C.byref(n)) != 0:
            raise R8bGpuError(_err())
        return int(z.value), int(n.value)


DEVICE_ALL, DEVICE_CURRENT = -1, -2
_host_allocs = {}


def host_free(arr):
    """Release an array from Batch.host_alloc()."""
    p = _host_allocs.pop(arr.ctypes.data, None)
    if p is not None:
        lib().r8bgpu_host_free(C.c_void_p(p))


class Batch:
    """n_channels independent streams resampled in lock-step: on one GPU (device >= 0, or DEVICE_CURRENT), or sharded
    over every visible GPU behind the C-ABI (DEVICE_ALL: host-buffer calls only).  Batch.mixed() makes a batch whose
    channels run different plans."""

    plans = None  # a mixed batch: its plans, and plan_of[c] = the index of channel c's plan
    plan_of = None
    _owner = None  # a part view (Batch.part): the mixed batch that owns the handle

    def __init__(self, plan, n_channels, device=-2):
        self.plan = plan
        self.n_channels = int(n_channels)
        self._h = lib().r8bgpu_batch_create(plan._h, self.n_channels, int(device))
        if not self._h:
            raise R8bGpuError(_err())

    @classmethod
    def mixed(cls, plans, plan_of, device=-2):
        """Independent streams at different rates in one batch: channel c runs plans[plan_of[c]] (r8bgpu_batch_create_mixed;
        the plans share one MaxInLen).  The ragged calls, clear_channels, flush, channel_totals and oneshot_clips work per
        channel; the lock-step calls and stage_kernels() raise (ask part(i) instead)."""
        plans = list(plans)
        po = np.ascontiguousarray(plan_of, dtype=np.int32).reshape(-1)
        hs = (C.c_void_p * len(plans))(*[p._h for p in plans])
        self = cls.__new__(cls)
        self.plan, self.plans, self.plan_of, self.n_channels = None, plans, po, len(po)
        self._h = lib().r8bgpu_batch_create_mixed(hs, len(plans), po.ctypes.data, len(po), int(device))
        if not self._h:
            raise R8bGpuError(_err())
        return self

    def part(self, i):
        """The ordinary batch behind plans[i] of a mixed batch (a view for introspection: stage_kernels(),
        kernel_launches, stage_times(); it lives as long as this batch)."""
        h = lib().r8bgpu_batch_part(self._h, int(i))
        if not h:
            raise R8bGpuError(_err())
        v = Batch.__new__(Batch)
        v.plan, v._h, v._owner = self.plans[int(i)], h, self
        v.n_channels = int(lib().r8bgpu_batch_channels(h))
        return v

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None and self._owner is None:
            _lib.r8bgpu_batch_destroy(self._h)
        self._h = None

    @property
    def max_out_len(self):
        """Room per channel a ragged call needs (a mixed batch: the largest of its plans')."""
        return int(lib().r8bgpu_batch_max_out_len(self._h))

    @property
    def flush_max_out_len(self):
        """Upper bound of what a default-target flush returns per channel (a mixed batch: the largest of its plans')."""
        return int(lib().r8bgpu_batch_flush_max_out_len(self._h))

    @property
    def max_in_len(self):
        return (self.plan or self.plans[0]).max_in_len

    def channel_plan(self, c):
        """The plan channel c runs."""
        return self.plan if self.plans is None else self.plans[int(self.plan_of[c])]

    def _refuse_lockstep(self):
        if self.plans is not None:  # the C-ABI refuses every lock-step call on a mixed batch; raise its message
            lib().r8bgpu_batch_process(self._h, None, 0, 0, None, 0, 0)
            raise R8bGpuError(_err())

    def shards(self):
        """[(device, first_channel, n_channels, numa_node)] -- one entry for a single-device batch."""
        out = []
        for i in range(lib().r8bgpu_batch_shard_count(self._h)):
            d, c0, n, node = C.c_int(0), C.c_int(0), C.c_int(0), C.c_int(0)
            if lib().r8bgpu_batch_shard_info(self._h, i, C.byref(d), C.byref(c0), C.byref(n), C.byref(node)) != 0:
                raise R8bGpuError(_err())
            out.append((d.value, c0.value, n.value, node.value))
        return out

    def host_alloc(self, samples_per_channel, dtype="float64"):
        """Pinned planar [n_channels, samples_per_channel] numpy array, rows on the NUMA node of the owning GPU.
        Keep the returned array alive while in use; release with host_free(arr)."""
        import numpy as np
        dt = np.dtype(dtype)
        p = lib().r8bgpu_batch_host_alloc(self._h, int(samples_per_channel), dt.itemsize)
        if not p:
            raise R8bGpuError(_err())
        n = self.n_channels * int(samples_per_channel)
        buf = (C.c_char * (n * dt.itemsize)).from_address(p)
        arr = np.frombuffer(buf, dtype=dt, count=n).reshape(self.n_channels, int(samples_per_channel))
        arr.flags.writeable = True
        _host_allocs[arr.ctypes.data] = p
        return arr

    def clear(self):
        if lib().r8bgpu_batch_clear(self._h) != 0:
            raise R8bGpuError(_err())

    def clear_channels(self, channels):
        """clear() on the named channels only: they restart as fresh resamplers, the others continue."""
        ch = np.ascontiguousarray(channels, dtype=np.int32).reshape(-1)
        if lib().r8bgpu_batch_clear_channels(self._h, ch.ctypes.data, len(ch)) != 0:
            raise R8bGpuError(_err())

    @property
    def channel_groups(self):
        """Distinct channel schedules (1: the channels run in lock-step)."""
        return int(lib().r8bgpu_batch_channel_groups(self._h))

    def set_trim(self, channels, factors):
        """Trim plans: channel channels[i] runs at dst * factors[i] from its next call on (r8bgpu_batch_set_trim).  The
        factors survive clear() and clear_channels()."""
        ch = np.ascontiguousarray(channels, dtype=np.int32).reshape(-1)
        fs = np.ascontiguousarray(factors, dtype=np.float64).reshape(-1)
        if len(fs) != len(ch):
            raise ValueError("expected one factor per channel named")
        if lib().r8bgpu_batch_set_trim(self._h, ch.ctypes.data, len(ch), fs.ctypes.data) != 0:
            raise R8bGpuError(_err())

    def trim(self):
        """Each channel's trim factor (1 for channels of an ordinary plan)."""
        fs = np.ones(self.n_channels, dtype=np.float64)
        if lib().r8bgpu_batch_trim(self._h, fs.ctypes.data) != 0:
            raise R8bGpuError(_err())
        return fs

    def set_dither(self, channels, seeds, taps=None, kind=DITHER_TPDF):
        """Dithered integer output for the named channels (r8bgpu_batch_set_dither): seeds is one seed or one per channel;
        taps None (flat TPDF), one list of error-feedback taps c_1.. for every channel, or one list per channel; kind
        DITHER_OFF restores the plain cast.  Settings survive clear(), clear_channels() and flushes."""
        ch = np.ascontiguousarray(channels, dtype=np.int64).reshape(-1)
        sd = np.broadcast_to(np.asarray(seeds, dtype=np.uint64), ch.shape)
        if taps is None or len(taps) == 0 or np.ndim(taps[0]) == 0:
            per = [taps] * len(ch)
        else:
            per = list(taps)
            if len(per) != len(ch):
                raise ValueError("expected one tap list per channel named")
        cfg = (Dither * max(len(ch), 1))(*[Dither.make(int(sd[i]), per[i], kind) for i in range(len(ch))])
        ci = ch.astype(np.int32)
        if lib().r8bgpu_batch_set_dither(self._h, ci.ctypes.data, len(ci), cfg) != 0:
            raise R8bGpuError(_err())

    def set_dsd_out(self, on=True):
        """One-bit DSD output (r8bgpu_batch_set_dsd_out): while on, the typed and flush calls take out_fmt=DSD_LSB /
        DSD_MSB only and return uint8 bytes, count / 8 per channel; counts are multiples of 8 samples.  Turning it on
        starts every channel's modulator afresh."""
        if lib().r8bgpu_batch_set_dsd_out(self._h, 1 if on else 0) != 0:
            raise R8bGpuError(_err())

    def dsd_overloads(self):
        """Each channel's modulator overloads since its last clear (int64 array)."""
        n = np.zeros(self.n_channels, dtype=np.int64)
        if lib().r8bgpu_batch_dsd_overloads(self._h, n.ctypes.data) != 0:
            raise R8bGpuError(_err())
        return n

    def _state_stride(self, ch):
        return max([self.channel_plan(int(c)).state_bytes for c in ch] + [8])

    def export_channels(self, channels, device=False):
        """The complete state of the named channels' streams (r8bgpu_batch_export): a list of bytes, one blob per channel,
        or with device=True a CUDA uint8 tensor [n, stride] on the batch's GPU (r8bgpu_batch_export_device; blob i in
        row i, its first Plan.state_bytes bytes).  Import a blob into any slot of a batch of the same plan and the stream
        continues there bit for bit.  Changes no output."""
        ch = np.ascontiguousarray(channels, dtype=np.int32).reshape(-1)
        stride = self._state_stride(ch)
        if device:
            import torch
            dev = torch.device("cuda", self.shards()[0][0])
            buf = torch.empty((len(ch), stride), dtype=torch.uint8, device=dev)
            self.set_stream(torch.cuda.current_stream(dev).cuda_stream)
            if lib().r8bgpu_batch_export_device(self._h, ch.ctypes.data, len(ch), buf.data_ptr(), stride) != 0:
                raise R8bGpuError(_err())
            return buf
        buf = np.zeros(len(ch) * stride, dtype=np.uint8)
        if lib().r8bgpu_batch_export(self._h, ch.ctypes.data, len(ch), buf.ctypes.data, stride) != 0:
            raise R8bGpuError(_err())
        return [buf[i * stride:i * stride + self.channel_plan(int(c)).state_bytes].tobytes() for i, c in enumerate(ch)]

    def import_channels(self, channels, states):
        """Channel channels[i] takes the stream of states[i] (r8bgpu_batch_import): a bytes-like blob from
        export_channels, or states is the CUDA uint8 tensor export_channels(device=True) returns (row i for channel i).
        Acts like clear_channels followed by installing the exported state; refused blobs change nothing."""
        ch = np.ascontiguousarray(channels, dtype=np.int32).reshape(-1)
        if hasattr(states, "is_cuda") and states.is_cuda:
            import torch
            if states.dtype != torch.uint8 or states.dim() != 2 or states.shape[0] != len(ch) or not states.is_contiguous():
                raise ValueError("expected a contiguous CUDA uint8 tensor [n_channels, stride]")
            self.set_stream(torch.cuda.current_stream(states.device).cuda_stream)
            rc = lib().r8bgpu_batch_import_device(self._h, ch.ctypes.data, len(ch), states.data_ptr(), states.shape[1])
        else:
            states = [bytes(s) for s in states]
            if len(states) != len(ch):
                raise ValueError("expected one state per channel named")
            stride = self._state_stride(ch)
            for i, (c, s) in enumerate(zip(ch, states)):
                want = self.channel_plan(int(c)).state_bytes
                if len(s) < want:
                    raise R8bGpuError("import_channels: channel %d: truncated blob (%d of %d bytes)" % (c, len(s), want))
            buf = np.zeros(len(ch) * stride, dtype=np.uint8)
            for i, s in enumerate(states):
                n = min(len(s), stride)
                buf[i * stride:i * stride + n] = np.frombuffer(s[:n], dtype=np.uint8)
            rc = lib().r8bgpu_batch_import(self._h, ch.ctypes.data, len(ch), buf.ctypes.data, stride)
        if rc != 0:
            raise R8bGpuError(_err())

    def process_ragged(self, xs):
        """One block per channel, each of its own length (0..MaxInLen): xs is a list of n_channels 1-D float64 numpy
        arrays (host path) or CUDA tensors (device path, on torch's current stream).  Returns the list of per-channel
        outputs, in the same kind."""
        if len(xs) != self.n_channels:
            raise ValueError("expected one block per channel")
        lens = np.array([len(x) for x in xs], dtype=np.int32)
        counts = np.empty(self.n_channels, dtype=np.int32)
        cap = max(self.max_out_len, 1)
        width = max(int(lens.max()), 1)
        if all(isinstance(x, np.ndarray) for x in xs):
            x = np.zeros((self.n_channels, width), dtype=np.float64)
            for c, xc in enumerate(xs):
                x[c, :len(xc)] = xc
            y = np.empty((self.n_channels, cap), dtype=np.float64)
            rc = lib().r8bgpu_batch_process_host_ragged(self._h, x.ctypes.data, width, lens.ctypes.data,
                                                        y.ctypes.data, cap, cap, counts.ctypes.data)
        else:
            import torch
            dev = xs[0].device
            x = torch.zeros((self.n_channels, width), dtype=torch.float64, device=dev)
            for c, xc in enumerate(xs):
                assert xc.is_cuda and xc.dtype == torch.float64 and xc.dim() == 1
                x[c, :len(xc)] = xc
            y = torch.empty((self.n_channels, cap), dtype=torch.float64, device=dev)
            self.set_stream(torch.cuda.current_stream(dev).cuda_stream)
            rc = lib().r8bgpu_batch_process_ragged(self._h, x.data_ptr(), width, lens.ctypes.data, y.data_ptr(), cap,
                                                   cap, counts.ctypes.data)
        if rc < 0:
            raise R8bGpuError(_err())
        return [y[c, :int(counts[c])] for c in range(self.n_channels)]

    def process_ragged_fmt(self, x, lens, out_dtype=None, interleaved=False, in_scale=1.0, out_scale=1.0, fmt=None,
                           out_fmt=None):
        """One block per channel, each of its own length lens[c] (0..MaxInLen), in a typed buffer: x is a padded planar
        [n_channels, width] array, or [width, n_channels] when interleaved -- a numpy array (host path) of
        int16/int32/float32/float64/uint8 (U8; fmt=ULAW / ALAW for G.711 bytes, fmt=DSD_LSB / DSD_MSB for DSD bytes of 8
        samples each, the width then counting bytes), or uint8 [..., 3] with fmt=S24, or a CUDA tensor (device path, on
        torch's current stream) of those types.  lens count samples.  Returns (y, counts): y in the same layout and kind,
        in out_dtype (default: the input's; float64 for DSD), padded with zeros to max_out_len; channel c's output is its
        first counts[c] samples (out_fmt=DSD_LSB / DSD_MSB, with DSD output on: uint8, its first counts[c] / 8 bytes)."""
        lens = np.ascontiguousarray(lens, dtype=np.int32).reshape(-1)
        if len(lens) != self.n_channels:
            raise ValueError("expected one length per channel")
        nch = self.n_channels
        width = x.shape[0] if interleaved else x.shape[1]
        if (x.shape[1] if interleaved else x.shape[0]) != nch:
            raise ValueError("channel count mismatch")
        if len(lens) and int(lens.max()) > width * FORMAT_SAMPLES.get(fmt, 1):
            raise ValueError("a length exceeds the buffer's width")
        cap = max(self.max_out_len, 1)
        counts = np.empty(nch, dtype=np.int32)
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x)
            fi = _NP_FORMATS[x.dtype.name] if fmt is None else fmt
            if out_fmt is None:
                out_fmt = _default_out(fi) if out_dtype is None else _NP_FORMATS[np.dtype(out_dtype).name]
            np_out = _NP_DTYPES[out_fmt]
            tail = (3,) if out_fmt == S24 else ()
            ce = max(_elems(out_fmt, cap), 1)
            y = np.zeros(((ce, nch) if interleaved else (nch, ce)) + tail, dtype=np_out)
            bi = Buffer.make(x.ctypes.data, fi, interleaved, nch if interleaved else width, in_scale)
            bo = Buffer.make(y.ctypes.data, out_fmt, interleaved, nch if interleaved else ce, out_scale)
            rc = lib().r8bgpu_batch_process_host_ragged_fmt(self._h, C.byref(bi), lens.ctypes.data, C.byref(bo), cap,
                                                            counts.ctypes.data)
        else:
            import torch
            th = {torch.float64: F64, torch.float32: F32, torch.int16: S16, torch.int32: S32, torch.uint8: U8}
            assert x.is_cuda
            x = x.contiguous()
            fi = th[x.dtype] if fmt is None else fmt
            if out_fmt is None:
                out_fmt = _default_out(fi) if out_dtype is None else th[out_dtype]
            t_out = {v: k for k, v in th.items()}.get(out_fmt, torch.uint8)
            tail = (3,) if out_fmt == S24 else ()
            ce = max(_elems(out_fmt, cap), 1)
            y = torch.zeros(((ce, nch) if interleaved else (nch, ce)) + tail, dtype=t_out, device=x.device)
            bi = Buffer.make(x.data_ptr(), fi, interleaved, nch if interleaved else width, in_scale)
            bo = Buffer.make(y.data_ptr(), out_fmt, interleaved, nch if interleaved else ce, out_scale)
            self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
            rc = lib().r8bgpu_batch_process_ragged_fmt(self._h, C.byref(bi), lens.ctypes.data, C.byref(bo), cap,
                                                       counts.ctypes.data)
        if rc < 0:
            raise R8bGpuError(_err())
        return y, counts

    def channel_totals(self):
        """(n_in, n_out): each channel's input and output sample totals since its last clear (int64 arrays)."""
        n_in = np.zeros(self.n_channels, dtype=np.int64)
        n_out = np.zeros(self.n_channels, dtype=np.int64)
        if lib().r8bgpu_batch_channel_totals(self._h, n_in.ctypes.data, n_out.ctypes.data) != 0:
            raise R8bGpuError(_err())
        return n_in, n_out

    def _out_buffer(self, cap, out_fmt, interleaved, device):
        """Zeroed output block [n_channels, cap] (interleaved: [cap, n_channels]; S24: trailing 3 bytes)."""
        nch = self.n_channels
        shape = ((cap, nch) if interleaved else (nch, cap)) + ((3,) if out_fmt == S24 else ())
        if device is None:
            return np.zeros(shape, dtype=_NP_DTYPES[out_fmt])
        import torch
        dt = getattr(torch, np.dtype(_NP_DTYPES[out_fmt]).name)
        return torch.zeros(shape, dtype=dt, device=device)

    def _flush_into(self, ch, tg, y, out_fmt, interleaved, out_scale, counts):
        cap = (y.shape[0] if interleaved else y.shape[1]) * FORMAT_SAMPLES.get(out_fmt, 1)
        host = isinstance(y, np.ndarray)
        bo = Buffer.make(y.ctypes.data if host else y.data_ptr(), out_fmt, interleaved,
                         self.n_channels if interleaved else _elems(out_fmt, cap), out_scale)
        if not host:
            import torch
            self.set_stream(torch.cuda.current_stream(y.device).cuda_stream)
        fn = lib().r8bgpu_batch_flush_host if host else lib().r8bgpu_batch_flush
        if fn(self._h, ch.ctypes.data, len(ch), None if tg is None else tg.ctypes.data, C.byref(bo), cap,
              counts.ctypes.data) < 0:
            raise R8bGpuError(_err())

    def flush(self, channels, targets=None, out_dtype=None, interleaved=False, device=None, out_scale=1.0, out_fmt=None):
        """End the named channels' streams (the silence-feeding tail of CDSPResampler::oneshot(), CDSPResampler.h:592-651):
        each is fed silence until its output since its last clear reaches its target (targets: absolute output counts;
        None: ceil(inputs * dst / src)), returns the samples up to the target, and is then cleared.  The other channels
        keep their state.  device: None / False for a host numpy result, or a CUDA device (torch.device or index) for a
        tensor there, produced on torch's current stream.  Returns (y, counts): y planar [n_channels, max(counts)] (or
        [max(counts), n_channels] when interleaved) in out_dtype (default float64; out_fmt=S24 gives packed uint8
        [..., 3]; out_fmt=DSD_LSB / DSD_MSB, with DSD output on, uint8 bytes of 8 samples), channel c's tail being its
        first counts[c] samples."""
        ch = np.ascontiguousarray(channels, dtype=np.int32).reshape(-1)
        tg = None if targets is None else np.ascontiguousarray(targets, dtype=np.int64).reshape(-1)
        if tg is not None and len(tg) != len(ch):
            raise ValueError("expected one target per channel named")
        cap = self.flush_max_out_len
        if tg is not None and len(ch) and ch.min() >= 0 and ch.max() < self.n_channels:
            cap = max(cap, int((tg - self.channel_totals()[1][ch]).max()))
        if out_fmt is None:
            out_fmt = F64 if out_dtype is None else _dtype_format(out_dtype)
        k = FORMAT_SAMPLES.get(out_fmt, 1)  # DSD: room for the held-back bits and the last byte's fill
        ce = max((cap + 2 * (k - 1)) // k if k > 1 else cap, 1)
        y = self._out_buffer(ce, out_fmt, interleaved, None if device is None or device is False else device)
        counts = np.zeros(self.n_channels, dtype=np.int32)
        self._flush_into(ch, tg, y, out_fmt, interleaved, out_scale, counts)
        m = _elems(out_fmt, int(counts.max())) if len(counts) else 0
        return (y[:m] if interleaved else y[:, :m]), counts

    def oneshot_clips(self, x, lens, oplens=None, out_dtype=None, interleaved=False, in_scale=1.0, out_scale=1.0,
                      fmt=None, out_fmt=None):
        """Resample a padded batch of whole clips, one per channel: per channel, what the reference's
        oneshot(ip, lens[c], op, oplens[c]) (CDSPResampler.h:592-651) returns on a fresh object.  x: planar
        [n_channels, width] (interleaved: [width, n_channels]), a numpy array (host path) or a CUDA tensor (device path,
        on torch's current stream), in the formats of process_ragged_fmt.  oplens default to ceil(lens * dst / src) of each
        channel's own plan.  lens count samples (DSD: 8 per byte of the width).
        Every channel is cleared first; clips longer than MaxInLen go in as several ragged calls (cut at multiples of 8
        samples for DSD), then one flush
        completes every clip.  The batch is left cleared.  Returns (y, oplens): y [n_channels, max(oplens)] (or
        interleaved) in out_dtype (default: the input's), zero past each clip's oplens[c]."""
        nch = self.n_channels
        lens = np.ascontiguousarray(lens, dtype=np.int64).reshape(-1)
        if len(lens) != nch or (x.shape[1] if interleaved else x.shape[0]) != nch:
            raise ValueError("expected one clip per channel")
        width = x.shape[0] if interleaved else x.shape[1]
        if len(lens) and (lens.min() < 0 or lens.max() > width * FORMAT_SAMPLES.get(fmt, 1)):
            raise ValueError("clip lengths must lie in [0, width]")
        if oplens is None:
            oplens = np.array([self.channel_plan(c).default_target(v) for c, v in enumerate(lens)], dtype=np.int64)
        oplens = np.ascontiguousarray(oplens, dtype=np.int64).reshape(-1)
        if len(oplens) != nch or (len(oplens) and oplens.min() < 0):
            raise ValueError("expected one non-negative output length per channel")
        host = isinstance(x, np.ndarray)
        if host:
            x = np.ascontiguousarray(x)
            fi = _NP_FORMATS[x.dtype.name] if fmt is None else fmt
            ptr, dev = x.ctypes.data, None
        else:
            import torch
            x = x.contiguous()
            fi = _dtype_format(x.dtype) if fmt is None else fmt
            ptr, dev = x.data_ptr(), x.device
            self.set_stream(torch.cuda.current_stream(dev).cuda_stream)
        if out_fmt is None:
            out_fmt = _default_out(fi) if out_dtype is None else _dtype_format(out_dtype)
        ein, spe = FORMAT_BYTES[fi], FORMAT_SAMPLES.get(fi, 1)
        W = max(int(oplens.max()) if nch else 0, 1)
        # the device form keeps one spare sample per channel past W: samples a block holds beyond a clip's end land there
        y = self._out_buffer(W if host else W + 1, out_fmt, interleaved, dev)
        pos = np.zeros(nch, dtype=np.int64)  # samples of each clip delivered so far

        def place(t, take):
            """Append the first take[c] samples of channel c of block t at pos[c] of y."""
            if host:
                for c in np.nonzero(take > 0)[0]:
                    k, p = int(take[c]), int(pos[c])
                    if interleaved:
                        y[p:p + k, c] = t[:k, c]
                    else:
                        y[c, p:p + k] = t[c, :k]
                return
            import torch
            ax = 0 if interleaved else 1
            j = torch.arange(t.shape[ax], device=dev)
            tk, ps = torch.as_tensor(take, device=dev), torch.as_tensor(pos, device=dev)
            if interleaved:
                idx = torch.where(j[:, None] < tk[None, :], j[:, None] + ps[None, :], W)
            else:
                idx = torch.where(j[None, :] < tk[:, None], j[None, :] + ps[:, None], W)
            if t.dim() == 3:  # packed 24-bit samples: 3 bytes each
                idx = idx[..., None].expand(-1, -1, 3)
            y.scatter_(ax, idx, t)

        self.clear()
        M = self.max_in_len - self.max_in_len % spe  # blocks of whole elements
        if M <= 0:
            raise ValueError("MaxInLen holds no whole element of this format")
        cap = max(self.max_out_len, 1)
        blk = self._out_buffer(cap, out_fmt, interleaved, dev)
        counts = np.zeros(nch, dtype=np.int32)
        fn = lib().r8bgpu_batch_process_host_ragged_fmt if host else lib().r8bgpu_batch_process_ragged_fmt
        for off in range(0, int(lens.max()) if nch else 0, M):
            ln = np.clip(lens - off, 0, M).astype(np.int32)
            bi = Buffer.make(ptr + off // spe * ein * (nch if interleaved else 1), fi, interleaved, nch if interleaved else width,
                             in_scale)
            bo = Buffer.make(blk.ctypes.data if host else blk.data_ptr(), out_fmt, interleaved, nch if interleaved else cap,
                             out_scale)
            if fn(self._h, C.byref(bi), ln.ctypes.data, C.byref(bo), cap, counts.ctypes.data) < 0:
                raise R8bGpuError(_err())
            take = np.minimum(counts, oplens - pos)
            place(blk, take)
            pos += take
        tail = self._out_buffer(max(int((oplens - pos).max()) if nch else 0, 1), out_fmt, interleaved, dev)
        self._flush_into(np.arange(nch, dtype=np.int32), oplens, tail, out_fmt, interleaved, out_scale, counts)
        place(tail, counts.astype(np.int64))
        if not host:
            y = y[:W] if interleaved else y[:, :W]
        return y, oplens

    def oneshot_long(self, x, lens=None, oplens=None, fmt=None, out_fmt=None, interleaved=False, in_scale=1.0, out_scale=1.0,
                     dither=None, plan_of=None):
        """Resample whole clips on every lane of the batch (r8bgpu_batch_oneshot / _oneshot_host): clip r's output is bit
        for bit what oneshot_clips returns for it on a one-channel batch of this plan, whatever the lane count.  x: planar
        [n_clips, width] (interleaved: [width, n_clips]; S24: [..., 3] uint8; DSD: bytes of 8 samples), a numpy array (host
        form) or a CUDA tensor (device form, on torch's current stream), in the formats of process_ragged_fmt.  lens: samples
        per clip (default: the width); oplens: output samples per clip (default ceil(lens * dst / src)).  dither: None, or
        one seed per clip (flat TPDF on integer outputs; None entries: off).  plan_of: None, or one plan index per clip
        (r8bgpu_batch_oneshot_mixed / _mixed_host): clip r runs self.plans[plan_of[r]] on that part's lanes, bit for bit
        as on an ordinary batch of that plan, and its default oplens are that plan's.  The batch is cleared before and
        after.  Returns (y, oplens): y [n_clips, max(oplens)] (or interleaved) in out_fmt (default: the input's; float64
        for DSD), zero past each clip's oplens[r]."""
        x, bi, fi, dev, lens, po = self._clips_in(x, lens, fmt, interleaved, in_scale, plan_of)
        n_clips = len(lens)
        oplens = self._clip_oplens(oplens, n_clips)
        if oplens is None:
            oplens = self._clip_targets(po, lens)
        y, bo = _rows_out(fi, out_fmt, dev, interleaved, n_clips, max(int(oplens.max()) if n_clips else 0, 1), out_scale)
        dv = _clip_dither(dither, n_clips)
        if po is None:
            fn = lib().r8bgpu_batch_oneshot_host if dev is None else lib().r8bgpu_batch_oneshot
            rc = fn(self._h, C.byref(bi), n_clips, lens.ctypes.data, C.byref(bo), oplens.ctypes.data, dv)
        else:
            fn = lib().r8bgpu_batch_oneshot_mixed_host if dev is None else lib().r8bgpu_batch_oneshot_mixed
            rc = fn(self._h, C.byref(bi), n_clips, po.ctypes.data, lens.ctypes.data, C.byref(bo), oplens.ctypes.data, dv)
        if rc != 0:
            raise R8bGpuError(_err())
        return y, oplens

    def oneshot_crops(self, x, crops, lens=None, oplens=None, fmt=None, out_fmt=None, interleaved=False, in_scale=1.0,
                      out_scale=1.0, dither=None, plan_of=None):
        """Crops of long clips (r8bgpu_batch_oneshot_crops / _crops_host): crops [n, 3] of (clip, o0, o1) ask for outputs
        [o0, o1) of the clip's oneshot_long output, and get exactly those bits, whatever else the call holds.  x, lens,
        oplens, formats, scales, dither (one seed per clip) and plan_of are those of oneshot_long.  Only the crops' spans
        of each clip run.  Returns y [n_crops, max(o1 - o0)] (interleaved: transposed) in out_fmt, zero past each crop's
        length."""
        x, bi, fi, dev, lens, po = self._clips_in(x, lens, fmt, interleaved, in_scale, plan_of)
        n_clips = len(lens)
        op = self._clip_oplens(oplens, n_clips)
        cr = _crops(crops)
        n = len(cr)
        y, bo = _rows_out(fi, out_fmt, dev, interleaved, n, max(int((cr["o1"] - cr["o0"]).max()) if n else 0, 1), out_scale)
        fn = lib().r8bgpu_batch_oneshot_crops_host if dev is None else lib().r8bgpu_batch_oneshot_crops
        rc = fn(self._h, C.byref(bi), n_clips, None if po is None else po.ctypes.data, lens.ctypes.data,
                None if op is None else op.ctypes.data, n, cr.ctypes.data if n else None, C.byref(bo),
                _clip_dither(dither, n_clips))
        if rc != 0:
            raise R8bGpuError(_err())
        return y

    def oneshot_crops_adjoint(self, gy, crops, lens, oplens=None, width=None, interleaved=False, plan_of=None):
        """The transpose of oneshot_crops (r8bgpu_batch_oneshot_crops_adjoint): gy (a float64 or float32 CUDA tensor
        [n_crops, W], W >= max(o1 - o0); interleaved: [W, n_crops]) holds each crop's output gradient.  Returns gx
        [n_clips, width] (width: default max(lens)) of gy's dtype: zeros, with each named clip's hull written, the sum of
        its crops' gradients in crop order."""
        gy, n_rows, W = _grad_in("oneshot_crops_adjoint", gy, interleaved)
        cr = _crops(crops)
        n = len(cr)
        if n_rows != n:
            raise ValueError("expected one gradient row per crop")
        lens = np.ascontiguousarray(lens, dtype=np.int64).reshape(-1)
        n_clips = len(lens)
        po = self._clip_plans(plan_of, n_clips)
        op = self._clip_oplens(oplens, n_clips)
        gx, bg, bx = self._grad_out(gy, n, W, lens, width, interleaved)
        rc = lib().r8bgpu_batch_oneshot_crops_adjoint(self._h, C.byref(bg), n_clips, None if po is None else po.ctypes.data,
                                                      lens.ctypes.data, None if op is None else op.ctypes.data, n,
                                                      cr.ctypes.data if n else None, C.byref(bx))
        if rc != 0:
            raise R8bGpuError(_err())
        return gx

    def _clips_in(self, x, lens, fmt, interleaved, in_scale, plan_of):
        """The input side of oneshot_long and oneshot_crops.  Returns (x, bi, fi, dev, lens, po): x contiguous (bi points
        into it), its buffer and format, dev (None: a host array; else the tensor's device, whose current stream the batch
        takes), lens (default: the width) and plan_of (_clip_plans)."""
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x)
            fi = _NP_FORMATS[x.dtype.name] if fmt is None else fmt
            ptr, dev = x.ctypes.data, None
        else:
            import torch
            x = x.contiguous()
            fi = _dtype_format(x.dtype) if fmt is None else fmt
            ptr, dev = x.data_ptr(), x.device
            self.set_stream(torch.cuda.current_stream(dev).cuda_stream)
        n_clips = x.shape[1] if interleaved else x.shape[0]
        width = x.shape[0] if interleaved else x.shape[1]
        spe = FORMAT_SAMPLES.get(fi, 1)
        lens = np.full(n_clips, width * spe, dtype=np.int64) if lens is None else np.ascontiguousarray(lens, dtype=np.int64)
        if len(lens) != n_clips:
            raise ValueError("expected one length per clip")
        if n_clips and (lens.min() < 0 or lens.max() > width * spe):
            raise ValueError("clip lengths must lie in [0, width]")
        po = self._clip_plans(plan_of, n_clips)
        return x, Buffer.make(ptr, fi, interleaved, n_clips if interleaved else width, in_scale), fi, dev, lens, po

    def _grad_out(self, gy, n_rows, W, lens, width, interleaved):
        """The input gradient of the adjoints: (gx, bg, bx), gx zeros [n_clips, width] (width: default max(lens)) of gy's
        dtype on torch's current stream, which the batch takes, and the buffers of gy (n_rows rows of W) and gx."""
        import torch
        n_clips = len(lens)
        width = max(int(lens.max()) if n_clips else 0, 1) if width is None else int(width)
        if n_clips and lens.max() > width:
            raise ValueError("width is smaller than the clip lengths")
        self.set_stream(torch.cuda.current_stream(gy.device).cuda_stream)
        fmt = _dtype_format(gy.dtype)
        gx = torch.zeros((width, n_clips) if interleaved else (n_clips, width), dtype=gy.dtype, device=gy.device)
        bg = Buffer.make(gy.data_ptr(), fmt, interleaved, max(n_rows, 1) if interleaved else W, 1.0)
        bx = Buffer.make(gx.data_ptr(), fmt, interleaved, n_clips if interleaved else width, 1.0)
        return gx, bg, bx

    def _clip_plans(self, plan_of, n_clips):
        """plan_of as an int32 array of one plan index per clip (None stays None)."""
        if plan_of is None:
            return None
        po = np.ascontiguousarray(plan_of, dtype=np.int32).reshape(-1)
        if len(po) != n_clips:
            raise ValueError("expected one plan index per clip")
        return po

    def _clip_oplens(self, oplens, n_clips):
        """oplens as an int64 array of one output length per clip (None stays None: the library's defaults)."""
        op = None if oplens is None else np.ascontiguousarray(oplens, dtype=np.int64).reshape(-1)
        if op is not None and len(op) != n_clips:
            raise ValueError("expected one output length per clip")
        return op

    def _clip_targets(self, po, lens):
        """Default output lengths: ceil(lens * dst / src) of each clip's plan (po None: the batch's first plan)."""
        nplans = len(self.plans) if self.plans is not None else 1

        def plan_of(r):
            if po is None:
                return self.channel_plan(0)
            p = int(po[r])
            if not 0 <= p < nplans:  # the C-ABI refuses it with its message
                return None
            return self.plan if self.plans is None else self.plans[p]
        tg = [plan_of(r) for r in range(len(lens))]
        return np.array([0 if pl is None else pl.default_target(int(v)) for pl, v in zip(tg, lens)], dtype=np.int64)

    def oneshot_adjoint(self, gy, lens=None, oplens=None, width=None, interleaved=False, plan_of=None):
        """The transpose of oneshot_long (r8bgpu_batch_oneshot_adjoint): for each clip r, the gradient of its lens[r]
        input samples from gy's row r, the gradient of its oplens[r] outputs.  gy: a float64 or float32 CUDA tensor
        [n_clips, W] (interleaved: [W, n_clips]), W >= max(oplens), on torch's current stream.  lens: the clips' input
        lengths (required: gy's width is an output length); oplens: default ceil(lens * dst / src).  plan_of: None, or one
        plan index per clip (r8bgpu_batch_oneshot_adjoint_mixed), as for oneshot_long.  Returns a tensor of gy's dtype and
        layout, [n_clips, width] (width: default max(lens)), zero past each lens[r]."""
        if lens is None:
            raise ValueError("oneshot_adjoint needs the clips' input lengths (lens)")
        gy, n_clips, W = _grad_in("oneshot_adjoint", gy, interleaved)
        lens = np.ascontiguousarray(lens, dtype=np.int64).reshape(-1)
        if len(lens) != n_clips:
            raise ValueError("expected one length per clip")
        po = self._clip_plans(plan_of, n_clips)
        oplens = self._clip_oplens(oplens, n_clips)
        if oplens is None:
            oplens = self._clip_targets(po, lens)
        if n_clips and oplens.max() > W:
            raise ValueError("gy is narrower than the output lengths")
        gx, bg, bx = self._grad_out(gy, n_clips, W, lens, width, interleaved)
        if po is None:
            rc = lib().r8bgpu_batch_oneshot_adjoint(self._h, C.byref(bg), n_clips, lens.ctypes.data, oplens.ctypes.data,
                                                    C.byref(bx))
        else:
            rc = lib().r8bgpu_batch_oneshot_adjoint_mixed(self._h, C.byref(bg), n_clips, po.ctypes.data, lens.ctypes.data,
                                                          oplens.ctypes.data, C.byref(bx))
        if rc != 0:
            raise R8bGpuError(_err())
        return gx

    def set_stream(self, cuda_stream_ptr):
        lib().r8bgpu_batch_set_stream(self._h, C.c_void_p(int(cuda_stream_ptr) if cuda_stream_ptr else None))

    def sync(self):
        if lib().r8bgpu_batch_sync(self._h) != 0:
            raise R8bGpuError(_err())

    @property
    def kernel_launches(self):
        return int(lib().r8bgpu_batch_kernel_launches(self._h))

    @property
    def device_bytes(self):
        return int(lib().r8bgpu_batch_device_bytes(self._h))

    def stage_kernels(self):
        """[(kernel_name, n_plan_stages_covered)] per plan stage."""
        if self.plans is not None:  # refused by the C-ABI: a stage index means nothing across plans
            lib().r8bgpu_batch_stage_kernel(self._h, 0, None, 0)
            raise R8bGpuError(_err())
        out = []
        for i in range(len(self.plan.stages())):
            buf = C.create_string_buffer(64)
            n = lib().r8bgpu_batch_stage_kernel(self._h, i, buf, 64)
            out.append((buf.value.decode(), n))
        return out

    def last_variant(self, stage):
        """The fused kernel's instantiation the last lock-step call launched for plan stage `stage` (its BlockConvolver),
        e.g. "k_up2_frac2<8,false,0,true,2,false,false,true,true> mbu=6", or the half-band cascade starting there with
        its tile plan, e.g. "k_hbup_cascade stages=5 taps=11/6/5/4/3 last2=1 w=160", or an unfused BlockConvolver or
        interpolator kernel with its call fields, e.g. "k_blockconv M=2048 up=2 src_up=1 down=3 trunc=0 tiles=6",
        "k_bcl M=65536 R0=16 src_up=1 down=1 trunc=0 tiles=2 groups=1" or "k_frac poly=1 tile=256 flen=24"; "" when
        none has."""
        n = lib().r8bgpu_batch_last_variant(self._h, int(stage), None, 0)
        if n < 0:
            raise R8bGpuError(_err())
        buf = C.create_string_buffer(n + 1)
        lib().r8bgpu_batch_last_variant(self._h, int(stage), buf, n + 1)
        return buf.value.decode()

    def set_timing(self, enable=True):
        lib().r8bgpu_batch_set_timing(self._h, int(bool(enable)))

    def stage_times(self):
        """[(stage_name, accumulated_ms, launches)] since set_timing(True); synchronises."""
        if self.plans is not None:  # refused by the C-ABI: a stage index means nothing across plans
            lib().r8bgpu_batch_stage_time_ms(self._h, 0, None)
            raise R8bGpuError(_err())
        out = []
        for i, st in enumerate(self.plan.stages()):
            n = C.c_ulonglong(0)
            ms = lib().r8bgpu_batch_stage_time_ms(self._h, i, C.byref(n))
            if ms < 0:
                raise R8bGpuError(_err())
            out.append((st["name"], ms, int(n.value)))
        return out

    def process_ptr(self, d_in, in_stride, l, d_out, out_stride, out_cap):
        """Raw device-pointer call (asynchronous).  Returns samples produced per channel."""
        self._refuse_lockstep()
        n = lib().r8bgpu_batch_process(self._h, C.c_void_p(int(d_in) if d_in else None), int(in_stride), int(l),
                                       C.c_void_p(int(d_out) if d_out else None), int(out_stride), int(out_cap))
        if n < 0:
            raise R8bGpuError(_err())
        return n

    def process_host_ptr(self, h_in, in_stride, l, h_out, out_stride, out_cap):
        self._refuse_lockstep()
        n = lib().r8bgpu_batch_process_host(self._h, C.c_void_p(int(h_in) if h_in else None), int(in_stride), int(l),
                                            C.c_void_p(int(h_out) if h_out else None), int(out_stride), int(out_cap))
        if n < 0:
            raise R8bGpuError(_err())
        return n

    def process_fmt(self, buf_in, l, buf_out, out_cap, host):
        """Typed buffers (Buffer.make(...)): host=True -> r8bgpu_batch_process_host_fmt, else device."""
        self._refuse_lockstep()
        fn = lib().r8bgpu_batch_process_host_fmt if host else lib().r8bgpu_batch_process_fmt
        n = fn(self._h, C.byref(buf_in), int(l), C.byref(buf_out), int(out_cap))
        if n < 0:
            raise R8bGpuError(_err())
        return n

    def process_host_fmt(self, x, out_dtype=None, interleaved=False, in_scale=1.0, out_scale=1.0, fmt=None,
                         out_fmt=None):
        """x: numpy array of int16/int32/float32/float64/uint8 (U8) samples, planar [n_channels, l] or (interleaved=True)
        [l, n_channels]; packed 24-bit is uint8 [..., 3] with fmt=S24, G.711 bytes are uint8 with fmt=ULAW / ALAW, DSD bytes
        (8 samples each: l = 8 * the width) are uint8 with fmt=DSD_LSB / DSD_MSB.
        Returns the same layout in out_dtype (default: the input's; float64 for DSD) -- the conversions of
        oneshot<Tin,Tout>() (CDSPResampler.h:592-651)."""
        self._refuse_lockstep()
        x = np.ascontiguousarray(x)
        fi = _NP_FORMATS[x.dtype.name] if fmt is None else fmt
        shape = x.shape[:2]
        w, nch = (shape[0], shape[1]) if interleaved else (shape[1], shape[0])
        l = w * FORMAT_SAMPLES.get(fi, 1)
        if nch != self.n_channels:
            raise ValueError("channel count mismatch")
        if out_fmt is None:
            out_fmt = _default_out(fi) if out_dtype is None else _NP_FORMATS[np.dtype(out_dtype).name]
        cap = max(self.max_out_len, 1)
        np_out = _NP_DTYPES[out_fmt]
        tail = (3,) if out_fmt == S24 else ()
        ce = max(_elems(out_fmt, cap), 1)  # DSD output: bytes
        y = np.empty(((ce, nch) if interleaved else (nch, ce)) + tail, dtype=np_out)
        bi = Buffer.make(x.ctypes.data, fi, interleaved, nch if interleaved else w, in_scale)
        bo = Buffer.make(y.ctypes.data, out_fmt, interleaved, nch if interleaved else ce, out_scale)
        n = _elems(out_fmt, self.process_fmt(bi, l, bo, cap, host=True))
        return (y[:n] if interleaved else y[:, :n]).copy()

    def process_host(self, x):
        """x: float64 numpy [n_channels, l] (C-contiguous rows).  Returns [n_channels, n_out]."""
        self._refuse_lockstep()
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.ndim != 2 or x.shape[0] != self.n_channels:
            raise ValueError("expected [n_channels, l]")
        cap = self.plan.max_out_len
        y = np.empty((self.n_channels, max(cap, 1)), dtype=np.float64)
        n = self.process_host_ptr(x.ctypes.data, x.shape[1], x.shape[1], y.ctypes.data, y.shape[1], cap)
        return y[:, :n].copy()

    def process(self, x, out=None):
        """x: CUDA float64 torch tensor [n_channels, l]; returns a view [n_channels, n_out] of `out`
        (allocated when None).  Runs on torch's current stream."""
        self._refuse_lockstep()
        import torch
        assert x.is_cuda and x.dtype == torch.float64 and x.dim() == 2 and x.shape[0] == self.n_channels
        assert x.stride(1) == 1
        cap = max(self.plan.max_out_len, 1)
        if out is None:
            out = torch.empty((self.n_channels, cap), dtype=torch.float64, device=x.device)
        assert out.stride(1) == 1 and out.shape[1] >= cap
        self.set_stream(torch.cuda.current_stream(x.device).cuda_stream)
        n = self.process_ptr(x.data_ptr(), x.stride(0), x.shape[1], out.data_ptr(), out.stride(0), out.shape[1])
        return out[:, :n]


def _resample_function():
    import torch

    class Resample(torch.autograd.Function):
        """Forward: Batch.oneshot_long (bit for bit the twin run), or with crops Batch.oneshot_crops (bit for bit slices of
        it).  Backward: Batch.oneshot_adjoint or Batch.oneshot_crops_adjoint, its exact transpose."""

        @staticmethod
        def forward(ctx, x, batch, crops, lens, oplens, plan_of):
            if crops is None:
                y, oplens = batch.oneshot_long(x, lens=lens, oplens=oplens, plan_of=plan_of)
            else:
                y = batch.oneshot_crops(x, crops, lens=lens, oplens=oplens, plan_of=plan_of)
            ctx.batch, ctx.crops, ctx.lens, ctx.oplens, ctx.width, ctx.plan_of = batch, crops, lens, oplens, x.shape[1], plan_of
            return y

        @staticmethod
        def backward(ctx, gy):
            kw = dict(oplens=ctx.oplens, width=ctx.width, plan_of=ctx.plan_of)
            if ctx.crops is None:
                gx = ctx.batch.oneshot_adjoint(gy, lens=ctx.lens, **kw)
            else:
                gx = ctx.batch.oneshot_crops_adjoint(gy, ctx.crops, ctx.lens, **kw)
            return gx, None, None, None, None, None

    return Resample


_RESAMPLE = None


def _resample(name, batch, x, crops, lens, oplens, plan_of):
    """resample_clips (crops None) and resample_crops: their arguments normalised, then the autograd function."""
    global _RESAMPLE
    import torch
    if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dim() != 2 or x.dtype not in (torch.float64, torch.float32):
        raise TypeError(name + " takes a float64 or float32 CUDA tensor [n_clips, T]")
    n_clips, T = x.shape
    lens = np.full(n_clips, T, dtype=np.int64) if lens is None else np.ascontiguousarray(lens, dtype=np.int64).reshape(-1)
    if oplens is not None:
        oplens = np.ascontiguousarray(oplens, dtype=np.int64).reshape(-1)
    if plan_of is not None:
        plan_of = np.ascontiguousarray(plan_of, dtype=np.int32).reshape(-1)
    if _RESAMPLE is None:
        _RESAMPLE = _resample_function()
    return _RESAMPLE.apply(x, batch, crops, lens, oplens, plan_of)


def resample_clips(batch, x, lens=None, oplens=None, plan_of=None):
    """Whole-clip resampling that torch autograd can differentiate: y = batch.oneshot_long(x, lens, oplens)[0], and
    y.backward() gives x the gradient Batch.oneshot_adjoint computes.  x: a float64 or float32 CUDA tensor [n_clips, T]
    (lens: default T for every clip; oplens: default ceil(lens * dst / src)).  plan_of: None, or one plan index per clip
    of a mixed batch (clips at several rates in one call; default oplens per clip's plan).  y: [n_clips, max(oplens)] of
    x's dtype, zero past each oplens[r]; x's gradient has x's dtype and is zero past each lens[r]."""
    return _resample("resample_clips", batch, x, None, lens, oplens, plan_of)


class ResamplerBatch:
    """Channel-batched counterpart of the loop in example.cpp:30-67 (host numpy in/out)."""

    def __init__(self, n_channels, src_rate, dst_rate, max_in_len, trans_band=2.0, atten=ATTEN_24,
                 device=-1, extfft=0):
        self.plan = Plan(src_rate, dst_rate, max_in_len, trans_band, atten, extfft=extfft)
        self.batch = Batch(self.plan, n_channels, device)

    def process(self, x):
        return self.batch.process_host(x)

    def clear(self):
        self.batch.clear()

    def getMaxOutLen(self, _max_in_len=0):
        return self.plan.max_out_len


class CDSPResampler:
    """Single-stream object with the reference's method names (host buffers, n_channels == 1)."""

    def __init__(self, SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand=2.0, ReqAtten=206.91,
                 device=-1, extfft=0):
        self.MaxInLen = int(aMaxInLen)
        self.plan = Plan(SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, ReqAtten, extfft=extfft)
        self.batch = Batch(self.plan, 1, device)

    def process(self, ip):
        """ip: 1-D float64 array of l <= MaxInLen samples; returns the produced samples."""
        ip = np.ascontiguousarray(ip, dtype=np.float64).reshape(1, -1)
        if self.plan.passthrough:
            return ip[0]  # the reference returns the input buffer itself (CDSPResampler.h:563-574)
        return self.batch.process_host(ip)[0]

    def clear(self):
        self.batch.clear()

    def getMaxOutLen(self, _max_in_len=0):
        return self.plan.max_out_len

    def getInLenBeforeOutPos(self, ReqOutPos):
        return self.plan.in_len_before_out_pos(ReqOutPos)

    def getInputRequiredForOutput(self, ReqOutSamples):
        return self.plan.input_required_for_output(ReqOutSamples)

    def getLatency(self):
        return 0

    def getLatencyFrac(self):
        return self.plan.latency_frac()

    def getInLenBeforeOutStart(self, ReqOutPos=0):
        """Feeds single zero samples until the output passes ReqOutPos, then clears
        (CDSPResampler.h:443-464); evaluated on the host scheduler, no kernels run."""
        n = 4096
        while True:
            cs = np.cumsum(self.plan.simulate([1] * n))
            hit = np.nonzero(cs > ReqOutPos)[0]
            if len(hit):
                return int(hit[0])
            n *= 2

    def oneshot(self, ip, oplen):
        """Resample a whole signal: feeds MaxInLen chunks, then zeros, until oplen samples exist
        (CDSPResampler.h:592-651).  Returns a float64 array of oplen samples."""
        ip = np.ascontiguousarray(ip, dtype=np.float64)
        out = np.empty(int(oplen), dtype=np.float64)
        got, pos = 0, 0
        zeros = None
        while got < oplen:
            if pos < len(ip):
                chunk = ip[pos:pos + self.MaxInLen]
                pos += len(chunk)
            else:
                if zeros is None:
                    zeros = np.zeros(self.MaxInLen)
                chunk = zeros
            y = self.process(chunk)
            w = min(len(y), oplen - got)
            out[got:got + w] = y[:w]
            got += w
        self.clear()
        return out


class CDSPResampler16(CDSPResampler):
    def __init__(self, SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand=2.0, **kw):
        super().__init__(SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, ATTEN_16, **kw)


class CDSPResampler16IR(CDSPResampler):
    def __init__(self, SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand=2.0, **kw):
        super().__init__(SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, ATTEN_16IR, **kw)


class CDSPResampler24(CDSPResampler):
    def __init__(self, SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand=2.0, **kw):
        super().__init__(SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, ATTEN_24, **kw)


def resample_crops(batch, x, crops, lens=None, oplens=None, plan_of=None):
    """Crops of whole-clip resampling that torch autograd can differentiate: y = batch.oneshot_crops(x, crops, lens,
    oplens), row k being outputs [o0, o1) of clip crops[k, 0]'s resample_clips output, and y.backward() gives x the
    gradient Batch.oneshot_crops_adjoint computes; only the crops' spans run, forward and backward.  x: a float64 or
    float32 CUDA tensor [n_clips, T]; crops: [n, 3] of (clip, o0, o1).  y: [n_crops, max(o1 - o0)] of x's dtype, zero past
    each crop's length."""
    return _resample("resample_crops", batch, x, np.ascontiguousarray(crops, dtype=np.int64).reshape(-1, 3), lens, oplens,
                     plan_of)
