"""ctypes binding of libojph_b200.so (the C-ABI in include/ojph_b200.h).

The product path loads the nvcc-built library that sits next to this file and fails loudly
when it is missing -- there is no CPU fallback.  (tests/ may hand `bind()` the SIMT-emulator
build of the same sources to check kernel logic without a GPU; that never happens here.)
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# OJB_LIB_PATH: another nvcc build of the same library (A/B of compile-time knobs); still no fallback of any kind
LIB_PATH = os.environ.get("OJB_LIB_PATH") or os.path.join(_HERE, "libojph_b200.so")


class Params(C.Structure):
    _fields_ = [
        ("width", C.c_uint32), ("height", C.c_uint32), ("off_x", C.c_uint32), ("off_y", C.c_uint32),
        ("tile_w", C.c_uint32), ("tile_h", C.c_uint32), ("tile_off_x", C.c_uint32), ("tile_off_y", C.c_uint32),
        ("num_comps", C.c_uint32), ("bit_depth", C.c_uint32 * 16), ("is_signed", C.c_uint32 * 16),
        ("dx", C.c_uint32 * 16), ("dy", C.c_uint32 * 16),
        ("num_decomps", C.c_uint32), ("block_w", C.c_uint32), ("block_h", C.c_uint32),
        ("num_precincts", C.c_uint32), ("precinct_w", C.c_uint32 * 33), ("precinct_h", C.c_uint32 * 33),
        ("reversible", C.c_uint32), ("color_transform", C.c_uint32), ("prog_order", C.c_uint32),
        ("qstep", C.c_float), ("qfactor", C.c_uint32), ("tlm", C.c_uint32), ("tilepart_div", C.c_uint32),
        ("planar", C.c_int32),
        ("coc_present", C.c_uint32 * 16), ("coc_reversible", C.c_uint32 * 16), ("coc_num_decomps", C.c_uint32 * 16),
        ("coc_block_w", C.c_uint32 * 16), ("coc_block_h", C.c_uint32 * 16),
        ("coc_num_precincts", C.c_uint32 * 16), ("coc_precinct_w", (C.c_uint32 * 33) * 16), ("coc_precinct_h", (C.c_uint32 * 33) * 16),
        ("nlt_all", C.c_uint32), ("nlt_comp", C.c_uint32 * 16), ("nlt_seq", C.c_uint32 * 16),
        ("profile", C.c_uint32),
        ("qcc_calls", C.c_uint32 * 16), ("qcc_qstep", C.c_float * 16), ("qcc_qstep_seq", C.c_uint32 * 16),
        ("qcc_qfactor", C.c_uint32 * 16), ("qcc_ctype", C.c_uint32 * 16), ("qcc_qfactor_seq", C.c_uint32 * 16),
        ("dfs_num_levels", C.c_uint32), ("dfs_type", C.c_uint32 * 32),
        ("atk_num_steps", C.c_uint32), ("atk_reversible", C.c_uint32), ("atk_K", C.c_float), ("atk_A", C.c_float * 8),
        ("atk_a", C.c_int32 * 8), ("atk_b", C.c_int32 * 8), ("atk_e", C.c_uint32 * 8),
    ]


class FrameInfo(C.Structure):
    _fields_ = [
        ("width", C.c_uint32), ("height", C.c_uint32), ("off_x", C.c_uint32), ("off_y", C.c_uint32),
        ("num_comps", C.c_uint32), ("bit_depth", C.c_uint32 * 16), ("is_signed", C.c_uint32 * 16),
        ("dx", C.c_uint32 * 16), ("dy", C.c_uint32 * 16), ("comp_w", C.c_uint32 * 16), ("comp_h", C.c_uint32 * 16),
        ("num_decomps", C.c_uint32), ("reversible", C.c_uint32), ("color_transform", C.c_uint32),
        ("num_tiles", C.c_uint32), ("nlt_type", C.c_uint32 * 16),
    ]


class CodingStyle(C.Structure):
    _fields_ = [
        ("num_decomps", C.c_uint32), ("reversible", C.c_uint32), ("color_transform", C.c_uint32),
        ("block_w", C.c_uint32), ("block_h", C.c_uint32), ("precinct_w", C.c_uint32 * 33), ("precinct_h", C.c_uint32 * 33),
        ("prog_order", C.c_uint32), ("num_layers", C.c_uint32), ("may_use_sop", C.c_uint32), ("use_eph", C.c_uint32),
        ("vertical_causality", C.c_uint32), ("tile_w", C.c_uint32), ("tile_h", C.c_uint32), ("tile_off_x", C.c_uint32),
        ("tile_off_y", C.c_uint32),
    ]


class DeviceImage(C.Structure):
    """ojb_device_image: sample (x, y) of component c at base[c] + y * row_pitch[c] + x * col_stride[c] * sample size"""
    _fields_ = [("base", C.c_void_p * 16), ("row_pitch", C.c_uint64 * 16), ("col_stride", C.c_uint32 * 16)]


class Comment(C.Structure):
    _fields_ = [("data", C.c_void_p), ("len", C.c_uint16), ("rcom", C.c_uint16)]


_QR = 64      # OJB_QUALITY_MAX_ROUNDS


class QualityInfo(C.Structure):
    """ojb_quality_info: the quality-target search of the last frame encoded with one"""
    _fields_ = [
        ("num_samples", C.c_uint64), ("limit", C.c_uint64), ("sse_lo", C.c_uint64), ("sse_hi", C.c_uint64),
        ("comp_sse", C.c_double * 16), ("num_comps", C.c_uint32), ("reached", C.c_uint32), ("rounds", C.c_uint32),
        ("pass_measured", C.c_uint32), ("round_key", C.c_uint64 * _QR), ("round_sse_lo", C.c_uint64 * _QR),
        ("round_sse_hi", C.c_uint64 * _QR), ("round_body", C.c_uint64 * _QR), ("pass_key", C.c_uint64),
        ("fail_key", C.c_uint64), ("pass_body", C.c_uint64), ("fail_body", C.c_uint64), ("fail_measured", C.c_uint32),
        ("pad", C.c_uint32), ("body0", C.c_uint64), ("model_round1", C.c_double), ("ms_candidates", C.c_float), ("ms_rounds", C.c_float),
        ("ms_final", C.c_float), ("pad2", C.c_float),
    ]


CB_ALLGATHER = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64)
CB_BCAST = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32)
CB_SENDRECV = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32)


class CommCallbacks(C.Structure):
    _fields_ = [("ctx", C.c_void_p), ("allgather", CB_ALLGATHER), ("bcast", CB_BCAST), ("send", CB_SENDRECV), ("recv", CB_SENDRECV)]


class BlockDesc(C.Structure):
    _fields_ = [
        ("sample_off", C.c_uint64), ("stride", C.c_uint32), ("w", C.c_uint32), ("h", C.c_uint32),
        ("missing_msbs", C.c_uint32), ("num_passes", C.c_uint32), ("len1", C.c_uint32), ("len2", C.c_uint32),
        ("byte_off", C.c_uint64), ("status", C.c_uint32), ("causal", C.c_uint32),
    ]


# every symbol include/ojph_b200.h declares: name -> (restype, argtypes)
_VP, _U32, _U64, _I = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
SYMBOLS = {
    "ojb_last_error": (C.c_char_p, []),
    "ojb_version": (C.c_char_p, []),
    "ojb_device_count": (_I, []),
    "ojb_set_device": (_I, [_I]),
    "ojb_params_default": (None, [C.POINTER(Params)]),
    "ojb_host_alloc": (_VP, [_U64]),
    "ojb_host_free": (None, [_VP]),
    "ojb_enc_create": (_VP, []),
    "ojb_enc_destroy": (None, [_VP]),
    "ojb_enc_configure": (_I, [_VP, C.POINTER(Params), _U32]),
    "ojb_enc_set_comments": (_I, [_VP, C.POINTER(Comment), _U32]),
    "ojb_marks_reference": (_I, []),
    "ojb_enc_marks": (None, [_VP, C.POINTER(C.c_float)]),
    "ojb_dec_marks": (None, [_VP, C.POINTER(C.c_float)]),
    "ojb_enc_encode_raster": (_I, [_VP, _U32, _VP, C.c_uint64, _VP, C.c_uint64, C.POINTER(C.c_uint64)]),
    "ojb_dec_decode_raster": (_I, [_VP, _U32, _VP, C.c_uint64, C.POINTER(C.c_uint64)]),
    "ojb_enc_exchange": (_VP, [_VP, _VP, C.POINTER(_U32)]),
    "ojb_enc_flush": (_I, [_VP, _VP, _U64, C.POINTER(_U64)]),
    "ojb_enc_encode_frame": (_I, [_VP, C.POINTER(_VP), C.POINTER(_U32), _VP, _U64, C.POINTER(_U64)]),
    "ojb_enc_device_plane": (_VP, [_VP, _U32]),
    "ojb_enc_upload_frame": (_I, [_VP, C.POINTER(_VP), C.POINTER(_U32)]),
    "ojb_enc_encode_resident": (_I, [_VP, _VP, _U64, C.POINTER(_U64), _I]),
    "ojb_enc_encode_device": (_I, [_VP, C.POINTER(DeviceImage), _VP, _VP, _U64, C.POINTER(_U64), _I]),
    "ojb_enc_kernel_launches": (_U32, [_VP]),
    "ojb_enc_num_blocks": (_U32, [_VP]),
    "ojb_enc_set_target_size": (_I, [_VP, _U64]),
    "ojb_enc_min_size": (_I, [_VP, C.POINTER(_U64)]),
    "ojb_enc_set_target_mse": (_I, [_VP, C.c_double]),
    "ojb_enc_transcode_headers": (_I, [_VP, _VP, _U64, _I, _U32]),
    "ojb_enc_transcode_headers_reduced": (_I, [_VP, _VP, _U64, _I, _U32, _U32, C.POINTER(FrameInfo)]),
    "ojb_enc_transcode": (_I, [_VP, _VP, _U64, _I, _VP, _U64, C.POINTER(_U64), _I]),
    "ojb_enc_quality_info": (_I, [_VP, C.POINTER(QualityInfo)]),
    "ojb_enc_rate_info": (_I, [_VP, C.POINTER(_U32), C.POINTER(_U32), _VP, _VP, _VP, _VP, C.POINTER(_U64), C.POINTER(C.c_float)]),
    "ojb_enc_timings": (None, [_VP, C.POINTER(C.c_float)]),
    "ojb_dec_timings": (None, [_VP, C.POINTER(C.c_float)]),
    "ojb_enc_read_band": (_I, [_VP, _U32, _U32, _U32, _U32, _VP, C.POINTER(_U32), C.POINTER(_U32)]),
    "ojb_enc_band_info": (_I, [_VP, _U32, _U32, _U32, _U32, C.POINTER(_U32), C.POINTER(C.c_float)]),
    "ojb_dec_create": (_VP, []),
    "ojb_dec_destroy": (None, [_VP]),
    "ojb_dec_enable_resilience": (_I, [_VP]),
    "ojb_dec_read_headers": (_I, [_VP, _VP, _U64, _U32, C.POINTER(FrameInfo)]),
    "ojb_dec_decode_frame": (_I, [_VP, C.POINTER(_VP), C.POINTER(_U32)]),
    "ojb_dec_decode_resident": (_I, [_VP]),
    "ojb_dec_restrict_input_resolution": (_I, [_VP, _U32, _U32, C.POINTER(FrameInfo)]),
    "ojb_dec_get_coding_style": (_I, [_VP, _U32, C.POINTER(CodingStyle)]),
    "ojb_dec_set_planar": (_I, [_VP, _I]),
    "ojb_dec_begin_pull": (_I, [_VP]),
    "ojb_dec_pull": (_VP, [_VP, C.POINTER(_U32)]),
    "ojb_dec_decode_device": (_I, [_VP, C.POINTER(DeviceImage), _VP]),
    "ojb_dec_device_plane": (_VP, [_VP, _U32]),
    "ojb_dec_use_device_codestream": (_I, [_VP, _VP]),
    "ojb_dec_read_headers_device": (_I, [_VP, _VP, _U64, _U32, C.POINTER(FrameInfo)]),
    "ojb_dec_mirror_bytes": (_U64, [_VP]),
    "ojb_dec_failed_blocks": (_U32, [_VP]),
    "ojb_dec_list_blocks": (_I, [_VP, C.POINTER(BlockDesc), _U32, C.POINTER(_U32)]),
    "ojb_dec_kernel_launches": (_U32, [_VP]),
    "ojb_dec_read_band": (_I, [_VP, _U32, _U32, _U32, _U32, _VP, C.POINTER(_U32), C.POINTER(_U32)]),
    "ojb_shard_unique_id": (_I, [_VP]),
    "ojb_shard_create_nccl": (_VP, [_U32, _U32, _VP]),
    "ojb_shard_create": (_VP, [_U32, _U32, C.POINTER(CommCallbacks)]),
    "ojb_shard_destroy": (None, [_VP]),
    "ojb_shard_last_error": (C.c_char_p, []),
    "ojb_shard_enc_configure": (_I, [_VP, C.POINTER(Params), _U32, _U32]),
    "ojb_shard_enc_encode": (_I, [_VP, C.POINTER(_VP), C.POINTER(_U32), _VP, _U64, C.POINTER(_U64)]),
    "ojb_shard_dec_decode": (_I, [_VP, _VP, _U64, _U32, _U32, C.POINTER(_VP), C.POINTER(_U32), C.POINTER(FrameInfo)]),
    "ojb_shard_enc_upload": (_I, [_VP, C.POINTER(_VP), C.POINTER(_U32)]),
    "ojb_shard_enc_encode_resident": (_I, [_VP, C.POINTER(_U64)]),
    "ojb_shard_device_codestream": (_VP, [_VP]),
    "ojb_shard_dec_decode_resident": (_I, [_VP, _VP, _U64, _U32, _U32, C.POINTER(FrameInfo)]),
    "ojb_shard_device_plane": (_VP, [_VP, _U32]),
    "ojb_shard_gatherv": (_I, [_VP, _VP, _U64, _U32, _VP, _U64, C.POINTER(_U64)]),
    "ojb_shard_set_partition": (_I, [_VP, _U32]),
    "ojb_shard_region_rows": (_U32, [_VP, _U32, C.POINTER(_U32), C.POINTER(_U32)]),
    "ojb_shard_timings": (None, [_VP, C.POINTER(C.c_float)]),
    "ojb_shard_rank": (_U32, [_VP]),
    "ojb_shard_world": (_U32, [_VP]),
    "ojb_encode_blocks": (_I, [_VP, _U64, C.POINTER(BlockDesc), _U32, _VP, _U64, C.POINTER(_U64)]),
    "ojb_decode_blocks": (_I, [_VP, _U64, C.POINTER(BlockDesc), _U32, _VP, _U64]),
}


def bind(path):
    """Load a build of the C-ABI and attach prototypes to every declared symbol."""
    lib = C.CDLL(path)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)      # AttributeError if the library does not export it
        fn.restype = res
        fn.argtypes = args
    return lib


_lib = None


def lib():
    """The product library.  Raises if the CUDA build is absent -- never falls back."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  openjph_b200 has no CPU fallback.")
        _lib = bind(LIB_PATH)
    return _lib
