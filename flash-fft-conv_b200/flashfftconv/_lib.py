"""ctypes binding of the bffc C ABI (include/bffc.h).  The shared library is built in-tree by
`__graft_entry__.build()` as `flash-fft-conv_b200/libbffc.so`.  There is deliberately no fallback:
if the library is missing or the device is not sm_90, every compute call raises."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), 'libbffc.so')

BFFC_DTYPE_BF16 = 0
BFFC_DTYPE_FP16 = 1
BFFC_DTYPE_FP32 = 2          # depthwise convolution only
BFFC_LAYOUT_BHL = 0
BFFC_LAYOUT_BLH = 1
BFFC_PLAN_DETERMINISTIC = 1      # bffc_plan_create_ex: dk_f summed in a fixed order

_lib = None

# name -> (restype, argtypes); must list every symbol declared in include/bffc.h
_c = ctypes
SYMBOLS = {
    'bffc_abi_version': (_c.c_int, []),
    'bffc_last_error': (_c.c_char_p, []),
    'bffc_supported': (_c.c_int, [_c.c_int, _c.c_int]),
    'bffc_plan_create': (_c.c_int, [_c.POINTER(_c.c_void_p), _c.c_int, _c.c_int]),
    'bffc_plan_create_ex': (_c.c_int, [_c.POINTER(_c.c_void_p), _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    'bffc_plan_destroy': (_c.c_int, [_c.c_void_p]),
    'bffc_fft_size': (_c.c_int, [_c.c_void_p]),
    'bffc_length_multiple': (_c.c_int, [_c.c_void_p]),
    'bffc_kf_pack': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_void_p]),
    'bffc_kf_pack_rfft': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_void_p]),
    'bffc_dkf_unpack': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_void_p]),
    'bffc_dkf_unpack_half': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_void_p]),
    'bffc_filter_workspace_bytes': (_c.c_size_t, [_c.c_void_p, _c.c_int]),
    'bffc_kf_from_filter': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int, _c.c_void_p, _c.c_int, _c.c_int, _c.c_void_p,
                                       _c.c_size_t, _c.c_void_p]),
    'bffc_dk_from_dkf': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_void_p, _c.c_size_t,
                                    _c.c_void_p]),
    'bffc_kf_from_filter_band': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int, _c.c_void_p, _c.c_int, _c.c_int, _c.c_int,
                                            _c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_dk_from_dkf_band': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_int, _c.c_void_p,
                                         _c.c_size_t, _c.c_void_p]),
    'bffc_kf_from_filter_lags': (_c.c_int, [_c.c_void_p, _c.c_void_p] + [_c.c_int] * 4
                                 + [_c.c_void_p, _c.c_int, _c.c_int, _c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_dk_from_dkf_lags': (_c.c_int, [_c.c_void_p] * 3 + [_c.c_int] * 5 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_workspace_bytes': (_c.c_size_t, [_c.c_void_p, _c.c_int, _c.c_int, _c.c_int]),
    'bffc_workspace_bytes_ex': (_c.c_size_t, [_c.c_void_p, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    'bffc_workspace_bytes_blocked': (_c.c_size_t, [_c.c_void_p] + [_c.c_int] * 6),
    'bffc_fwd': (_c.c_int, [_c.c_void_p] * 6 + [_c.c_int] * 3 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_bwd': (_c.c_int, [_c.c_void_p] * 11 + [_c.c_int] * 3 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_fwd_strided': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_void_p, _c.c_int64,
                                    _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64] + [_c.c_int] * 3
                         + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_bwd_strided': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64, _c.c_void_p,
                                    _c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64, _c.c_void_p,
                                    _c.c_int64, _c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64]
                         + [_c.c_int] * 3 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_fwd_blocked': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_void_p, _c.c_int64,
                                    _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64] + [_c.c_int] * 4
                         + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_bwd_blocked': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64, _c.c_void_p,
                                    _c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64, _c.c_void_p,
                                    _c.c_int64, _c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64]
                         + [_c.c_int] * 4 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_fwd_short_strided': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_void_p, _c.c_int64,
                                          _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64] + [_c.c_int] * 3
                               + [_c.c_void_p] * 6 + [_c.c_int] * 3 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_bwd_short_strided': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64, _c.c_void_p,
                                          _c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64, _c.c_void_p,
                                          _c.c_int64, _c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64]
                               + [_c.c_int] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 3
                               + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_workspace_bytes_grouped': (_c.c_size_t, [_c.c_void_p] + [_c.c_int] * 7),
    'bffc_fwd_grouped': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_void_p, _c.c_int64,
                                    _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64] + [_c.c_int] * 5
                         + [_c.c_void_p] * 6 + [_c.c_int] * 3 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_bwd_grouped': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64, _c.c_void_p,
                                    _c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64, _c.c_void_p,
                                    _c.c_int64, _c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int64]
                         + [_c.c_int] * 5 + [_c.c_void_p] * 6 + [_c.c_int] * 3
                         + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_host_chunk_batch': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_int, _c.c_int]),
    'bffc_host_workspace_bytes': (_c.c_size_t, [_c.c_void_p, _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    'bffc_fwd_host': (_c.c_int, [_c.c_void_p] * 6 + [_c.c_int] * 3 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_last_launch_count': (_c.c_int, []),
    'bffc_dwconv1d_fwd': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_void_p]
                          + [_c.c_int] * 6 + [_c.c_void_p]),
    'bffc_dwconv1d_workspace_bytes': (_c.c_size_t, [_c.c_int] * 6),
    'bffc_dwconv1d_bwd': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int, _c.c_void_p, _c.c_int, _c.c_void_p, _c.c_void_p,
                                     _c.c_void_p] + [_c.c_int] * 6 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_dwconv1d_fwd_varlen': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_void_p]
                                 + [_c.c_int] * 6 + [_c.c_void_p, _c.c_int, _c.c_void_p]),
    'bffc_dwconv1d_bwd_varlen': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int, _c.c_void_p, _c.c_int, _c.c_void_p,
                                            _c.c_void_p, _c.c_void_p] + [_c.c_int] * 6
                                 + [_c.c_void_p, _c.c_int, _c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_conv_state_bytes': (_c.c_size_t, [_c.c_int] * 6),
    'bffc_conv_step_workspace_bytes': (_c.c_size_t, [_c.c_int] * 5),
    'bffc_conv_state_fill': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 9
                             + [_c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_void_p]),
    'bffc_conv_step': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p, _c.c_int] * 2 + [_c.c_void_p] * 6
                       + [_c.c_int] * 4 + [_c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_void_p, _c.c_int64]
                       + [_c.c_int] * 4 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_conv_step_slots_workspace_bytes': (_c.c_size_t, [_c.c_int] * 5),
    'bffc_conv_state_fill_slots': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 8
                                   + [_c.c_void_p] * 2 + [_c.c_int] * 2
                                   + [_c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_void_p]),
    'bffc_conv_step_slots': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p, _c.c_int] * 2 + [_c.c_void_p] * 6
                             + [_c.c_int] * 4 + [_c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_void_p, _c.c_int64]
                             + [_c.c_int] * 4 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_conv_far_layout': (_c.c_int, [_c.c_int] * 5 + [_c.POINTER(_c.c_int), _c.POINTER(_c.c_int),
                                                         _c.POINTER(_c.c_size_t)]),
    'bffc_conv_far_gather': (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_void_p] + [_c.c_int] * 8
                             + [_c.c_void_p] * 3),
    'bffc_conv_far_gather_slots': (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_void_p, _c.c_void_p]
                                   + [_c.c_int] * 9 + [_c.c_void_p] * 3),
    'bffc_conv_step_far': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p, _c.c_int] * 2 + [_c.c_void_p] * 6
                           + [_c.c_int] * 4 + [_c.c_void_p, _c.c_size_t] + [_c.c_void_p] * 5 + [_c.c_int64]
                           + [_c.c_int] * 4 + [_c.c_void_p]),
    'bffc_conv_step_far_slots': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p, _c.c_int] * 2
                                 + [_c.c_void_p] * 6 + [_c.c_int] * 4 + [_c.c_void_p, _c.c_size_t]
                                 + [_c.c_void_p] * 5 + [_c.c_int64] + [_c.c_int] * 4 + [_c.c_void_p]),
    'bffc_conv_extend_layout': (_c.c_int, [_c.c_int] * 7 + [_c.POINTER(_c.c_int), _c.POINTER(_c.c_int),
                                                            _c.POINTER(_c.c_size_t)]),
    'bffc_conv_extend_workspace_bytes': (_c.c_size_t, [_c.c_int] * 3),
    'bffc_conv_extend_gather': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 4
                                + [_c.c_void_p, _c.c_size_t, _c.c_void_p] + [_c.c_int] * 8
                                + [_c.c_void_p] * 3 + [_c.c_size_t, _c.c_void_p]),
    'bffc_conv_extend_gather_slots': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 4
                                      + [_c.c_void_p, _c.c_size_t, _c.c_void_p] + [_c.c_void_p] * 2 + [_c.c_int] * 9
                                      + [_c.c_void_p] * 3 + [_c.c_size_t, _c.c_void_p]),
    'bffc_conv_extend_finish': (_c.c_int, [_c.c_void_p] * 2 + [_c.c_int] * 2 + [_c.c_void_p] * 5 + [_c.c_int64]
                                + [_c.c_int] * 6 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_conv_extend_finish_slots': (_c.c_int, [_c.c_void_p] * 2 + [_c.c_int] * 2 + [_c.c_void_p] * 5 + [_c.c_int64]
                                      + [_c.c_int] * 7 + [_c.c_void_p, _c.c_size_t, _c.c_void_p]),
    'bffc_modal_fwd': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_int64, _c.c_void_p, _c.c_void_p]),
    'bffc_modal_workspace_bytes': (_c.c_size_t, [_c.c_int] * 3 + [_c.c_int64, _c.c_int]),
    'bffc_modal_bwd': (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_int64] + [_c.c_void_p] * 4
                       + [_c.c_size_t, _c.c_void_p]),
    'bffc_modal_transpose': (_c.c_int, [_c.c_void_p, _c.c_int64] + [_c.c_int] * 3 + [_c.c_int64, _c.c_void_p, _c.c_int]
                             + [_c.c_void_p] * 2 + [_c.c_int] * 2 + [_c.c_void_p] * 3 + [_c.c_int, _c.c_void_p,
                                                                                           _c.c_size_t, _c.c_void_p]),
    'bffc_modal_chunk': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 4
                         + [_c.c_void_p] * 2 + [_c.c_int] + [_c.c_void_p] * 2 + [_c.c_int] * 5 + [_c.c_void_p] * 3),
    'bffc_modal_step': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 4
                        + [_c.c_void_p] * 4 + [_c.c_int] * 2 + [_c.c_void_p, _c.c_int, _c.c_void_p, _c.c_int64]
                        + [_c.c_int] * 3 + [_c.c_void_p]),
    'bffc_modal_extend_finish': (_c.c_int, [_c.c_void_p] * 5 + [_c.c_int] * 3 + [_c.c_void_p, _c.c_int]
                                 + [_c.c_void_p] * 2 + [_c.c_int] * 4 + [_c.c_void_p, _c.c_int64, _c.c_void_p]),
    'bffc_fir_fwd': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] + [_c.c_int] * 4 + [_c.c_int64, _c.c_int]
                     + [_c.c_void_p, _c.c_int64, _c.c_void_p]),
    'bffc_fir_workspace_bytes': (_c.c_size_t, [_c.c_int, _c.c_int, _c.c_int64, _c.c_int]),
    'bffc_fir_bwd': (_c.c_int, [_c.c_void_p, _c.c_int64] * 4 + [_c.c_void_p] + [_c.c_int] * 4 + [_c.c_int64, _c.c_int]
                     + [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 2 + [_c.c_size_t, _c.c_void_p]),
    'bffc_fir_fwd_varlen': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] + [_c.c_int] * 4
                            + [_c.c_int64, _c.c_int] + [_c.c_void_p, _c.c_int64, _c.c_void_p, _c.c_int, _c.c_int64,
                                                        _c.c_void_p]),
    'bffc_fir_bwd_varlen': (_c.c_int, [_c.c_void_p, _c.c_int64] * 4 + [_c.c_void_p] + [_c.c_int] * 4
                            + [_c.c_int64, _c.c_int] + [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 2
                            + [_c.c_size_t, _c.c_void_p, _c.c_int, _c.c_int64, _c.c_void_p]),
    'bffc_fir_decode_state_bytes': (_c.c_size_t, [_c.c_int] * 5),
    'bffc_fir_decode_row_len': (_c.c_int64, [_c.c_int] * 2),
    'bffc_fir_decode_step': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 4
                             + [_c.c_void_p, _c.c_int, _c.c_int, _c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_int,
                                _c.c_void_p, _c.c_int64] + [_c.c_int] * 3 + [_c.c_void_p]),
    'bffc_fir_decode_gather': (_c.c_int, [_c.c_void_p, _c.c_int64] * 3 + [_c.c_void_p] * 6 + [_c.c_int] * 5
                               + [_c.c_void_p, _c.c_size_t, _c.c_void_p, _c.c_int] + [_c.c_void_p] * 2 + [_c.c_int] * 5
                               + [_c.c_void_p] * 4),
    'bffc_fir_decode_finish': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_int, _c.c_void_p, _c.c_int] + [_c.c_void_p] * 2
                               + [_c.c_int] * 5 + [_c.c_void_p, _c.c_int64, _c.c_void_p]),
    'bffc_docs_gather':(_c.c_int, [_c.c_void_p, _c.c_int, _c.c_int64] + [_c.c_int] * 3
                         + [_c.POINTER(_c.c_void_p), _c.POINTER(_c.c_int64), _c.POINTER(_c.c_void_p), _c.c_int,
                            _c.c_void_p]),
    'bffc_docs_scatter': (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_int64] + [_c.c_int] * 3
                          + [_c.POINTER(_c.c_void_p), _c.POINTER(_c.c_void_p), _c.POINTER(_c.c_int64), _c.c_int,
                             _c.c_void_p]),
}


class BffcError(RuntimeError):
    pass


def lib():
    """Load libbffc.so (once).  Raises BffcError loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise BffcError(f'{LIB_PATH} not found: run `python -c "import __graft_entry__ as g; g.build()"` '
                            'at the repo root (nvcc, sm_90a). There is no CPU/PyTorch fallback.')
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc):
    if rc != 0:
        raise BffcError(f'bffc error {rc}: {lib().bffc_last_error().decode()}')
