"""ctypes binding of libgccnmf_b200.so (the C ABI declared in include/gccnmf_b200.h).

PyTorch is used only as the device container (allocation, streams); every numeric op on the hot
path is one of the library's sm_90a kernels.  There is NO CPU fallback: importing this module
without the built library, or creating a handle without a CUDA device, raises.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libgccnmf_b200.so')


class GCCNMFError(RuntimeError):
    """A C-ABI call returned a negative status."""


class ParameterError(Exception):
    """Mirror of gccNMF/librosaSTFT.py:292-294 (mal-formed inputs)."""


GCCNMF_OK = 0
GCCNMF_ERR_INVALID_ARGUMENT = -1
GCCNMF_ERR_CUDA = -2
GCCNMF_ERR_WORKSPACE = -3
GCCNMF_ERR_UNSUPPORTED = -4
GCCNMF_ERR_NO_DEVICE = -5

_H = c_void_p   # gccnmf_handle*
_P = c_void_p   # device pointer
_S = c_void_p   # cudaStream_t

# name -> (restype, argtypes); must list every symbol of include/gccnmf_b200.h (tests check this)
SIGNATURES = {
    'gccnmf_abi_version': (c_int, []),
    'gccnmf_create': (c_int, [ctypes.POINTER(c_void_p), c_int]),
    'gccnmf_destroy': (c_int, [_H]),
    'gccnmf_last_error': (c_char_p, [_H]),
    'gccnmf_status_string': (c_char_p, [c_int]),
    'gccnmf_launch_count': (c_int64, [_H]),
    'gccnmf_set_option': (c_int, [_H, c_char_p, c_int]),
    'gccnmf_stft_num_frames': (c_int, [c_int64, c_int, c_int]),
    'gccnmf_stft': (c_int, [_H, _P, c_int64, c_int, c_int64, _P, c_int, c_int, c_int, _P, _P, _S]),
    'gccnmf_istft_length': (c_int64, [c_int, c_int, c_int, c_int]),
    'gccnmf_istft_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'gccnmf_istft_ola': (c_int, [_H, _P, c_int, c_int, c_int, c_int, _P, c_float, c_int, c_int, _P, _P, c_size_t, _S]),
    'gccnmf_klnmf_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'gccnmf_klnmf_uses_tensor_cores': (c_int, [_H, c_int, c_int, c_int]),
    'gccnmf_klnmf': (c_int, [_H, _P, c_int, c_int, _P, _P, c_int, c_int, c_float, c_float, c_int, _P, c_size_t, _S]),
    'gccnmf_klnmf_batched_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'gccnmf_klnmf_batched': (c_int, [_H, _P, c_int64, c_int64, c_int, c_int, c_int, _P, _P, c_int, c_int, c_float, c_float, c_int, _P, c_size_t, _S]),
    'gccnmf_klnmf_ragged_workspace_bytes': (c_size_t, [c_int, c_int, _P, c_int]),
    'gccnmf_klnmf_ragged': (c_int, [_H, _P, _P, _P, c_int, c_int, _P, _P, c_int, c_int, c_float, c_float, c_int, _P, c_size_t, _S]),
    'gccnmf_klnmf_begin': (c_int, [_H, _P, c_int, c_int, _P, _P, c_int, _P, c_size_t, _S]),
    'gccnmf_klnmf_step_numer': (c_int, [_H, _P, c_int, c_int, _P, _P, c_int, c_float, c_float, c_int, _P, _P, c_size_t, _S]),
    'gccnmf_klnmf_step_apply': (c_int, [_H, c_int, c_int, _P, _P, c_int, _P, _P, c_size_t, _S]),
    'gccnmf_klnmf_step_apply_multimem': (c_int, [_H, c_int, c_int, _P, _P, c_int, _P, _P, c_size_t, _S]),
    'gccnmf_klnmf_step_multimem': (c_int, [_H, _P, c_int, c_int, _P, _P, c_int, c_float, c_float, c_int, _P, _P, _P, _P, ctypes.c_uint32, _P, c_size_t, _S]),
    'gccnmf_klnmf_pull_buffer_floats': (c_int64, [c_int, c_int, c_int]),
    'gccnmf_klnmf_pull_supported': (c_int, [_H, c_int, c_int, c_int]),
    'gccnmf_klnmf_step_pull': (c_int, [_H, _P, c_int, c_int, _P, _P, c_int, c_float, c_float, c_int, c_int64, c_int, c_int, ctypes.POINTER(ctypes.c_void_p), c_int, c_int,
                                       c_int, _P, c_size_t, _S]),
    'gccnmf_klnmf_step_multimem2': (c_int, [_H, _P, c_int, c_int, _P, _P, c_int, c_float, c_float, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P,
                                            ctypes.c_uint32, _P, c_size_t, _S]),
    'gccnmf_klnmf_end': (c_int, [_H, c_int, c_int, _P, _P, c_int, c_int, _P, c_size_t, _S]),
    'gccnmf_phat_angspec_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'gccnmf_phat_angspec': (c_int, [_H, _P, c_int, c_int, c_int, _P, c_int, _P, _P, _P, _P, c_size_t, _S]),
    'gccnmf_tdoa_gccnmf': (c_int, [_H, _P, c_int, c_int, _P, c_int, _P, c_int, _P, _P, _S]),
    'gccnmf_tdoa_argmax_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'gccnmf_tdoa_argmax_refine_capacity': (c_int, [c_int, c_int]),
    'gccnmf_tdoa_argmax': (c_int, [_H, _P, c_int, c_int, _P, c_int, _P, c_int, _P, _P, _P, c_size_t, _S]),
    'gccnmf_coeff_mask': (c_int, [_H, _P, c_int, c_int, c_int, _P, _P, _S]),
    'gccnmf_argmax_mask': (c_int, [_H, _P, c_int, c_int, _P, c_int, _P, _S]),
    'gccnmf_online_targets': (c_int, [_H, _P, c_int, c_int, _P, _P, _S]),
    'gccnmf_atom_mask': (c_int, [_H, _P, c_int, c_int, _P, c_float, c_float, c_int, c_float, c_float, _P, _S]),
    'gccnmf_wiener_apply_workspace_bytes': (c_size_t, [c_int]),
    'gccnmf_wiener_apply': (c_int, [_H, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P, c_size_t, _S]),
    'gccnmf_masked_recon_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'gccnmf_masked_recon_phase': (c_int, [_H, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, c_size_t, _S]),
    'gccnmf_debug_timing': (c_int64, [_H, _P, c_int]),
    'gccnmf_klnmf_tile_plan': (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(c_int)]),
    'gccnmf_gemm_planes_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'gccnmf_gemm_planes': (c_int, [_H, _P, c_int, _P, c_int, _P, c_int, c_int, c_int, c_int, c_int, _P, c_size_t, _P, _S]),
}



class RtConfig(ctypes.Structure):
    """gccnmf_rt_config (include/gccnmf_b200.h)."""
    _fields_ = [('window_size', c_int), ('hop_size', c_int), ('block_size', c_int), ('windows_per_block', c_int), ('num_atoms', c_int),
                ('num_tdoas', c_int), ('history_length', c_int), ('inference_iterations', c_int), ('sparsity_alpha', c_float),
                ('epsilon', c_float)]


class PipelineConfig(ctypes.Structure):
    """gccnmf_pipeline_config (include/gccnmf_b200.h)."""
    _fields_ = [('window_size', c_int), ('hop_size', c_int), ('num_tdoas', c_int), ('num_atoms', c_int), ('num_iterations', c_int),
                ('num_targets', c_int), ('sparsity_alpha', c_float), ('epsilon', c_float), ('target_window_seconds', c_float)]


_C = ctypes.POINTER(RtConfig)
_PC = ctypes.POINTER(PipelineConfig)
SIGNATURES.update({
    'gccnmf_pipeline_workspace_bytes': (c_size_t, [_PC, c_int64]),
    'gccnmf_pick_targets': (c_int, [_H, _P, c_int, c_int, _P, _P, _S]),
    'gccnmf_separate': (c_int, [_H, _PC, _P, c_int64, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_size_t, _S]),
    'gccnmf_window_targets': (c_int, [_H, _P, c_int, c_int, c_int, c_int, _P, _P, _P, _S]),
    'gccnmf_target_gccnmf': (c_int, [_H, _P, c_int, c_int, _P, c_int, _P, c_int, _P, c_int, _P, _S]),
    'gccnmf_argmax_mask_frames': (c_int, [_H, _P, c_int, c_int, _P, c_int, _P, c_double, _P, _P, _S]),
    'gccnmf_pipeline_tracked_workspace_bytes': (c_size_t, [_PC, c_int, c_int64]),
    'gccnmf_separate_tracked': (c_int, [_H, _PC, c_int, _P, c_int64, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_size_t, _S]),
    'gccnmf_wiener_apply_h': (c_int, [_H, _P, _P, _P, _P, c_int, c_int, c_int, _P, _P, _S]),
    'gccnmf_rt_state_bytes': (c_size_t, [_C]),
    'gccnmf_rt_init': (c_int, [_H, _C, _P, _P, _P, _P, _P, _P, c_size_t, _S]),
    'gccnmf_rt_set_params': (c_int, [_H, _C, _P, c_size_t, c_float, c_int, c_float, c_float, c_float, c_int, c_int, c_int, c_int, _S]),
    'gccnmf_rt_process_frames': (c_int, [_H, _C, _P, c_size_t, _P, _P, _P, _S]),
    'gccnmf_rt_process_block': (c_int, [_H, _C, _P, c_size_t, _P, _P, _P, _S]),
    'gccnmf_rt_graph_create': (c_int, [_H, _C, _P, c_size_t, _P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_rt_graph_launch': (c_int, [_H, c_void_p, _S]),
    'gccnmf_rt_graph_destroy': (c_int, [_H, c_void_p]),
    'gccnmf_rt_export': (c_int, [_H, _C, _P, c_size_t, c_int, c_void_p, _S]),
})


class RtmSlotParams(ctypes.Structure):
    """gccnmf_rtm_slot_params (include/gccnmf_b200.h)."""
    _fields_ = [('target_index', c_float), ('set_target', c_int), ('epsilon', c_float), ('beta', c_float), ('noise_floor', c_float),
                ('mode', c_int), ('separation_enabled', c_int), ('localization_enabled', c_int), ('localization_window', c_int),
                ('active', c_int)]


SIGNATURES.update({
    'gccnmf_rtm_state_bytes': (c_size_t, [_C, c_int]),
    'gccnmf_rtm_init': (c_int, [_H, _C, c_int, _P, _P, _P, _P, _P, _P, c_size_t, _S]),
    'gccnmf_rtm_reset_slots': (c_int, [_H, _C, c_int, _P, c_size_t, c_int, c_int, _S]),
    'gccnmf_rtm_set_params': (c_int, [_H, _C, c_int, _P, c_size_t, c_int, c_int, ctypes.POINTER(RtmSlotParams), _S]),
    'gccnmf_rtm_process_frames': (c_int, [_H, _C, c_int, _P, c_size_t, _P, _P, _P, _S]),
    'gccnmf_rtm_process_block': (c_int, [_H, _C, c_int, _P, c_size_t, _P, _P, _P, _S]),
    'gccnmf_rtm_graph_create': (c_int, [_H, _C, c_int, _P, c_size_t, _P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_rtm_export': (c_int, [_H, _C, c_int, _P, c_size_t, c_int, c_int, c_void_p, _S]),
    'gccnmf_rtsep_state_bytes': (c_size_t, [_C, c_int, c_int]),
    'gccnmf_rtsep_init': (c_int, [_H, _C, c_int, c_int, _P, _P, _P, _P, _P, _P, c_size_t, _S]),
    'gccnmf_rtsep_reset_slots': (c_int, [_H, _C, c_int, c_int, _P, c_size_t, c_int, c_int, _S]),
    'gccnmf_rtsep_set_params': (c_int, [_H, _C, c_int, c_int, _P, c_size_t, c_int, c_int, ctypes.POINTER(RtmSlotParams), _S]),
    'gccnmf_rtsep_set_targets': (c_int, [_H, _C, c_int, c_int, _P, c_size_t, c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_rtsep_process_frames': (c_int, [_H, _C, c_int, c_int, _P, c_size_t, _P, _P, _S]),
    'gccnmf_rtsep_process_block': (c_int, [_H, _C, c_int, c_int, _P, c_size_t, _P, _P, _S]),
    'gccnmf_rtsep_graph_create': (c_int, [_H, _C, c_int, c_int, _P, c_size_t, _P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_rtsep_export': (c_int, [_H, _C, c_int, c_int, _P, c_size_t, c_int, c_int, c_void_p, _S]),
})

_PP = ctypes.POINTER(c_void_p)   # host array of device pointers
_BANK = [_H, _C, c_int, c_int, c_int, c_int, _P, c_size_t]     # h, cfg, S, P, Qd, Qe, state, state_bytes
SIGNATURES.update({
    'gccnmf_rtbank_state_bytes': (c_size_t, [_C, c_int, c_int, c_int, c_int]),
    'gccnmf_rtbank_init': (c_int, _BANK + [_PP, ctypes.POINTER(c_int), _PP, _PP, _P, _P, _S]),
    'gccnmf_rtbank_load_dictionary': (c_int, _BANK + [c_int, _P, c_int, _P, _S]),
    'gccnmf_rtbank_load_steering': (c_int, _BANK + [c_int, _P, _S]),
    'gccnmf_rtbank_assign': (c_int, _BANK + [c_int, c_int, ctypes.POINTER(c_int32), ctypes.POINTER(c_int32), _S]),
    'gccnmf_rtbank_reset_slots': (c_int, _BANK + [c_int, c_int, _S]),
    'gccnmf_rtbank_set_params': (c_int, _BANK + [c_int, c_int, ctypes.POINTER(RtmSlotParams), _S]),
    'gccnmf_rtbank_set_targets': (c_int, _BANK + [c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_rtbank_process_frames': (c_int, _BANK + [_P, _P, _P, _S]),
    'gccnmf_rtbank_process_block': (c_int, _BANK + [_P, _P, _P, _S]),
    'gccnmf_rtbank_graph_create': (c_int, _BANK + [_P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_rtbank_export': (c_int, _BANK + [c_int, c_int, c_void_p, _S]),
})

class LLConfig(ctypes.Structure):
    """gccnmf_ll_config (include/gccnmf_b200.h)."""
    _fields_ = [('window_size', c_int), ('hop_size', c_int), ('hops_per_call', c_int), ('num_atoms', c_int), ('num_tdoas', c_int),
                ('num_streams', c_int), ('inference_iterations', c_int), ('sparsity_alpha', c_float), ('epsilon', c_float)]


class LLStreamParams(ctypes.Structure):
    """gccnmf_ll_stream_params (include/gccnmf_b200.h)."""
    _fields_ = [('epsilon', c_float), ('active', c_int), ('target_override', c_int)]


_LC = ctypes.POINTER(LLConfig)
SIGNATURES.update({
    'gccnmf_ll_state_bytes': (c_size_t, [_LC]),
    'gccnmf_ll_init': (c_int, [_H, _LC, _P, _P, _P, _P, c_float, _P, _P, c_size_t, _S]),
    'gccnmf_ll_reset_streams': (c_int, [_H, _LC, _P, c_size_t, c_int, c_int, _S]),
    'gccnmf_ll_set_params': (c_int, [_H, _LC, _P, c_size_t, c_int, c_int, ctypes.POINTER(LLStreamParams), _S]),
    'gccnmf_ll_process': (c_int, [_H, _LC, _P, c_size_t, c_int, _P, _P, _S]),
    'gccnmf_ll_graph_create': (c_int, [_H, _LC, _P, c_size_t, c_int, _P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_ll_export': (c_int, [_H, _LC, _P, c_size_t, c_int, c_int, c_void_p, _S]),
    'gccnmf_llsep_state_bytes': (c_size_t, [_LC, c_int]),
    'gccnmf_llsep_init': (c_int, [_H, _LC, c_int, _P, _P, _P, _P, c_float, _P, _P, c_size_t, _S]),
    'gccnmf_llsep_reset_streams': (c_int, [_H, _LC, c_int, _P, c_size_t, c_int, c_int, _S]),
    'gccnmf_llsep_set_params': (c_int, [_H, _LC, c_int, _P, c_size_t, c_int, c_int, ctypes.POINTER(LLStreamParams), _S]),
    'gccnmf_llsep_set_targets': (c_int, [_H, _LC, c_int, _P, c_size_t, c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_llsep_process': (c_int, [_H, _LC, c_int, _P, c_size_t, c_int, _P, _P, _S]),
    'gccnmf_llsep_graph_create': (c_int, [_H, _LC, c_int, _P, c_size_t, c_int, _P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_llsep_export': (c_int, [_H, _LC, c_int, _P, c_size_t, c_int, c_int, c_void_p, _S]),
    'gccnmf_llrec_record_bytes': (c_size_t, [_LC, c_int]),
    'gccnmf_llrec_workspace_bytes': (c_size_t, [_LC, c_int, c_int]),
    'gccnmf_llrec_save_streams': (c_int, [_H, _LC, c_int, _P, c_size_t, c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
    'gccnmf_llrec_load_streams': (c_int, [_H, _LC, c_int, _P, c_size_t, c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
})

_HIST = [_H, _LC, c_int, c_int, _P, c_size_t]      # handle, config, num_sources, history_length, state, state_bytes
SIGNATURES.update({
    'gccnmf_llhist_state_bytes': (c_size_t, [_LC, c_int, c_int]),
    'gccnmf_llhist_init': (c_int, [_H, _LC, c_int, c_int, _P, _P, _P, _P, c_float, _P, _P, c_size_t, _S]),
    'gccnmf_llhist_reset_streams': (c_int, _HIST + [c_int, c_int, _S]),
    'gccnmf_llhist_set_params': (c_int, _HIST + [c_int, c_int, ctypes.POINTER(LLStreamParams), _S]),
    'gccnmf_llhist_set_targets': (c_int, _HIST + [c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_llhist_set_window': (c_int, _HIST + [c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_llhist_process': (c_int, _HIST + [c_int, _P, _P, _S]),
    'gccnmf_llhist_graph_create': (c_int, _HIST + [c_int, _P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_llhist_export': (c_int, _HIST + [c_int, c_int, c_void_p, _S]),
    'gccnmf_llhist_record_bytes': (c_size_t, [_LC, c_int, c_int]),
    'gccnmf_llhist_workspace_bytes': (c_size_t, [_LC, c_int, c_int, c_int]),
    'gccnmf_llhist_save_streams': (c_int, _HIST + [c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
    'gccnmf_llhist_load_streams': (c_int, _HIST + [c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
})
LLHIST_MAX_HISTORY = 1024
LLHIST_RECORD_CONFIG_HISTORY = 9        # config[9] of a record header: the history length (0 without history)


class RecordHeader(ctypes.Structure):
    """gccnmf_record_header (include/gccnmf_b200.h): the first bytes of every stream record."""
    _fields_ = [('magic', ctypes.c_uint32), ('abi_version', c_int32), ('kind', c_int32), ('num_sources', c_int32),
                ('payload_bytes', ctypes.c_uint64), ('synthesis_digest', ctypes.c_uint64), ('config', c_int32 * 16)]


RECORD_MAGIC = 0x52534347
RECORD_KIND_LL = 2
RECORD_HEADER_BYTES = 256

SIGNATURES.update({
    'gccnmf_rtrec_record_bytes': (c_size_t, [_C, c_int]),
    'gccnmf_rtrec_workspace_bytes': (c_size_t, [_C, c_int, c_int, c_int, c_int, c_int]),
    'gccnmf_rtrec_save_slots': (c_int, _BANK + [c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
    'gccnmf_rtrec_load_slots': (c_int, _BANK + [c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
})


class RtRecordHeader(ctypes.Structure):
    """gccnmf_rtrec_header (include/gccnmf_b200.h): the header of a real-time slot's record; its first 24 bytes are those of
    RecordHeader."""
    _fields_ = [('magic', ctypes.c_uint32), ('abi_version', c_int32), ('kind', c_int32), ('num_sources', c_int32),
                ('payload_bytes', ctypes.c_uint64), ('windows_digest', ctypes.c_uint64), ('dictionary_digest', ctypes.c_uint64),
                ('steering_digest', ctypes.c_uint64), ('dictionary_atoms', c_int32), ('reserved', c_int32), ('config', c_int32 * 16)]


RECORD_KIND_RT = 1
RTREC_DIGEST_CHUNK_WORDS = 1024

_LLBANK = [_H, _LC, c_int, c_int, c_int, _P, c_size_t]      # handle, config, num_sources, history_length, num_steerings, state, state_bytes
SIGNATURES.update({
    'gccnmf_llbank_state_bytes': (c_size_t, [_LC, c_int, c_int, c_int]),
    'gccnmf_llbank_init': (c_int, [_H, _LC, c_int, c_int, c_int, _P, _P, _P, _P, c_float, _P, _P, c_size_t, _S]),
    'gccnmf_llbank_load_steering': (c_int, _LLBANK + [c_int, _P, _S]),
    'gccnmf_llbank_assign': (c_int, _LLBANK + [c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_llbank_reset_streams': (c_int, _LLBANK + [c_int, c_int, _S]),
    'gccnmf_llbank_set_params': (c_int, _LLBANK + [c_int, c_int, ctypes.POINTER(LLStreamParams), _S]),
    'gccnmf_llbank_set_targets': (c_int, _LLBANK + [c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_llbank_set_window': (c_int, _LLBANK + [c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_llbank_process': (c_int, _LLBANK + [c_int, _P, _P, _S]),
    'gccnmf_llbank_graph_create': (c_int, _LLBANK + [c_int, _P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_llbank_export': (c_int, _LLBANK + [c_int, c_int, c_void_p, _S]),
    'gccnmf_llbank_record_bytes': (c_size_t, [_LC, c_int, c_int, c_int]),
    'gccnmf_llbank_workspace_bytes': (c_size_t, [_LC, c_int, c_int, c_int, c_int]),
    'gccnmf_llbank_save_streams': (c_int, _LLBANK + [c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
    'gccnmf_llbank_load_streams': (c_int, _LLBANK + [c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
})
LLBANK_MAX_STEERINGS = 64
RECORD_KIND_LLBANK = 3


_LLDICT = [_H, _LC, c_int, c_int, c_int, c_int, _P, c_size_t]   # handle, config, num_sources, history_length, num_dictionaries, num_steerings, state, state_bytes
SIGNATURES.update({
    'gccnmf_lldict_state_bytes': (c_size_t, [_LC, c_int, c_int, c_int, c_int]),
    'gccnmf_lldict_init': (c_int, [_H, _LC, c_int, c_int, c_int, c_int, ctypes.POINTER(c_void_p), ctypes.POINTER(c_int), ctypes.POINTER(c_void_p),
                                   _P, _P, _P, c_float, _P, c_size_t, _S]),
    'gccnmf_lldict_load_dictionary': (c_int, _LLDICT + [c_int, _P, c_int, _P, _S]),
    'gccnmf_lldict_load_steering': (c_int, _LLDICT + [c_int, _P, _S]),
    'gccnmf_lldict_assign': (c_int, _LLDICT + [c_int, c_int, ctypes.POINTER(c_int32), ctypes.POINTER(c_int32), _S]),
    'gccnmf_lldict_reset_streams': (c_int, _LLDICT + [c_int, c_int, _S]),
    'gccnmf_lldict_set_params': (c_int, _LLDICT + [c_int, c_int, ctypes.POINTER(LLStreamParams), _S]),
    'gccnmf_lldict_set_targets': (c_int, _LLDICT + [c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_lldict_set_window': (c_int, _LLDICT + [c_int, c_int, ctypes.POINTER(c_int32), _S]),
    'gccnmf_lldict_process': (c_int, _LLDICT + [c_int, _P, _P, _S]),
    'gccnmf_lldict_graph_create': (c_int, _LLDICT + [c_int, _P, _P, _P, _P, ctypes.POINTER(c_void_p), _S]),
    'gccnmf_lldict_export': (c_int, _LLDICT + [c_int, c_int, c_void_p, _S]),
    'gccnmf_lldict_record_bytes': (c_size_t, [_LC, c_int, c_int, c_int, c_int]),
    'gccnmf_lldict_workspace_bytes': (c_size_t, [_LC, c_int, c_int, c_int, c_int, c_int]),
    'gccnmf_lldict_save_streams': (c_int, _LLDICT + [c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
    'gccnmf_lldict_load_streams': (c_int, _LLDICT + [c_int, c_int, c_void_p, c_size_t, _P, c_size_t, _S]),
})
LLDICT_MAX_DICTIONARIES = 64


class LLBankRecordHeader(ctypes.Structure):
    """gccnmf_llbank_record_header (include/gccnmf_b200.h): RecordHeader's fields, then the content digests of the dictionary and of
    the stream's steering table."""
    _fields_ = RecordHeader._fields_ + [('dictionary_digest', ctypes.c_uint64), ('steering_digest', ctypes.c_uint64)]


_lib = None


def load_library():
    """dlopen the in-tree library and declare every signature.  Raises if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError('%s is missing: run `python -c "import __graft_entry__ as g; g.build()"` '
                          '(or python gcc-nmf_b200/build.py).  There is no CPU fallback.' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def _key_owner(key):
    while isinstance(key, tuple) and len(key) > 0:
        key = key[0]
    return key


def _ptr(t):
    """Device pointer of a torch tensor (None or empty -> NULL)."""
    if t is None or t.numel() == 0:
        return None
    assert t.is_cuda and t.is_contiguous(), 'device-resident contiguous tensor required'
    return t.data_ptr()


class Handle(object):
    """Owns one gccnmf_handle bound to a CUDA device; all methods enqueue on torch's current stream."""

    def __init__(self, device=0):
        import torch
        self.torch = torch
        self.lib = load_library()
        if not torch.cuda.is_available():
            raise GCCNMFError('no CUDA device visible: gcc-nmf_b200 has no CPU fallback')
        self.device = torch.device('cuda', device if isinstance(device, int) else torch.device(device).index or 0)
        torch.cuda.set_device(self.device)
        torch.zeros(1, device=self.device)   # make sure the primary context exists before the library binds to it
        h = c_void_p()
        st = self.lib.gccnmf_create(ctypes.byref(h), self.device.index)
        if st != GCCNMF_OK:
            raise GCCNMFError('gccnmf_create failed (%s): %s' % (self.lib.gccnmf_status_string(st).decode(),
                                                                 self.lib.gccnmf_last_error(None).decode()))
        self.h = h
        self._workspaces = {}
        self._buffers = {}

    def close(self):
        if getattr(self, 'h', None):
            self.lib.gccnmf_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ plumbing
    @property
    def stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    @property
    def launches(self):
        return int(self.lib.gccnmf_launch_count(self.h))

    def check(self, status):
        if status == GCCNMF_OK:
            return
        msg = self.lib.gccnmf_last_error(self.h).decode()
        if status == GCCNMF_ERR_INVALID_ARGUMENT:
            raise ParameterError(msg)
        raise GCCNMFError('%s: %s' % (self.lib.gccnmf_status_string(status).decode(), msg))

    def set_option(self, name, value):
        self.check(self.lib.gccnmf_set_option(self.h, name.encode(), int(value)))

    def klnmf_uses_tensor_cores(self, F, T2, K):
        return bool(self.lib.gccnmf_klnmf_uses_tensor_cores(self.h, F, T2, K))

    def workspace(self, key, nbytes):
        """Caller-owned scratch, cached per purpose and grown on demand."""
        ws = self._workspaces.get(key)
        if ws is None or ws.numel() < nbytes:
            ws = self.torch.empty(max(int(nbytes), 256), dtype=self.torch.uint8, device=self.device)
            self._workspaces[key] = ws
        return ws

    def empty(self, shape, dtype):
        return self.torch.empty(shape, dtype=dtype, device=self.device)

    def buffer(self, key, shape, dtype):
        """Persistent device buffer per key: allocated once (plan time) and reused by every later call with the same shape, so
        steady-state pipelines never enter the allocator (a cudaMalloc costs milliseconds).  A call with another shape REPLACES
        the buffer of that key (clips of varying length do not accumulate one buffer set per length)."""
        shape = tuple(int(v) for v in shape)
        entry = self._buffers.get(key)
        if entry is None or entry[0] != shape or entry[1] != dtype:
            entry = self._buffers[key] = (shape, dtype, self.torch.empty(shape, dtype=dtype, device=self.device))
        return entry[2]

    def release(self, owner):
        """Drops every persistent buffer whose key starts with `owner` (a pipeline's token; called when it is collected)."""
        for key in [k for k in self._buffers if k == owner or (isinstance(k, tuple) and len(k) > 0 and _key_owner(k) is owner)]:
            del self._buffers[key]

    def _out(self, out_key, name, shape, dtype):
        return self.empty(shape, dtype) if out_key is None else self.buffer((out_key, name), shape, dtype)

    def to_device(self, array, dtype=None):
        t = self.torch.as_tensor(array)
        if dtype is not None:
            t = t.to(dtype)
        return t.contiguous().to(self.device, non_blocking=True)

    # ------------------------------------------------------------------ ops (device tensors in / out)
    def stft(self, samples, window, n_fft, hop, conjugate=True, want_V=False, out_key=None, out=None):
        """samples (C, n) f32 cuda, window (n_fft) f64 cuda -> X (C, F, T) c64 [, V (F, C*T) f32].  out: (X, V) to write into
        (contiguous, of those shapes; V may be None)."""
        torch = self.torch
        C, n = samples.shape
        T = self.lib.gccnmf_stft_num_frames(n, n_fft, hop)
        if T < 1:
            if hop < 1:
                raise ParameterError('Invalid hop_length: %d' % hop)
            raise ParameterError('Buffer is too short (n=%d) for frame_length=%d' % (n, n_fft))
        F = n_fft // 2 + 1
        if out is not None:
            X, V = out
            if tuple(X.shape) != (C, F, T) or (V is not None and tuple(V.shape) != (F, C * T)):
                raise ParameterError('stft: out shapes %s do not match (%d, %d, %d)' % ([tuple(t.shape) for t in out if t is not None], C, F, T))
        else:
            X = self._out(out_key, 'X', (C, F, T), torch.complex64)
            V = self._out(out_key, 'V', (F, C * T), torch.float32) if want_V else None
        self.check(self.lib.gccnmf_stft(self.h, _ptr(samples), samples.stride(0), C, n, _ptr(window), n_fft, hop,
                                        1 if conjugate else 0, _ptr(X), _ptr(V), self.stream))
        return (X, V) if want_V else X

    def istft_ola(self, spec, window, n_fft, hop, gain=1.0, center=True, conjugate=True, out_key=None):
        """spec (B, F, T) c64 cuda -> y (B, length) f32."""
        torch = self.torch
        B, F, T = spec.shape
        length = self.lib.gccnmf_istft_length(n_fft, hop, T, 1 if center else 0)
        y = self._out(out_key, 'y', (B, max(int(length), 0)), torch.float32)
        nbytes = self.lib.gccnmf_istft_workspace_bytes(B, n_fft, T)
        ws = self.workspace('istft', nbytes)
        self.check(self.lib.gccnmf_istft_ola(self.h, _ptr(spec), B, n_fft, hop, T, _ptr(window), float(gain),
                                             1 if center else 0, 1 if conjugate else 0, _ptr(y), _ptr(ws), ws.numel(),
                                             self.stream))
        return y

    def klnmf(self, V, W, H, iterations, sparsity_alpha=0.0, epsilon=1e-16, update_W=True):
        """In place on W (F, K), H (K, T2) f32 cuda."""
        F, T2 = V.shape
        K = W.shape[1]
        ws = self.workspace('klnmf', self.lib.gccnmf_klnmf_workspace_bytes(F, T2, K))
        self.check(self.lib.gccnmf_klnmf(self.h, _ptr(V), F, T2, _ptr(W), _ptr(H), K, int(iterations),
                                         float(sparsity_alpha), float(epsilon), 1 if update_W else 0, _ptr(ws),
                                         ws.numel(), self.stream))
        return W, H

    def klnmf_batched(self, V, W, H, iterations, sparsity_alpha=0.0, epsilon=1e-16, update_W=True):
        """B clips in one call, in place on W (B, F, K), H (B, K, T2) f32 cuda.  V (B, F, T2) f32 cuda may be a strided view
        (unit stride along T2), e.g. clips side by side in the columns of one (F, B T2) matrix, read in place.  Clip b ends bit-identical to klnmf on it alone."""
        B, F, T2 = V.shape
        K = W.shape[2]
        if V.stride(2) != 1 or not V.is_cuda:
            raise ParameterError('klnmf_batched: V must be a cuda tensor with unit stride along T2')
        if tuple(W.shape) != (B, F, K) or tuple(H.shape) != (B, K, T2):
            raise ParameterError('klnmf_batched: W %s / H %s do not match V %s' % (tuple(W.shape), tuple(H.shape), tuple(V.shape)))
        ws = self.workspace('klnmf_batched', self.lib.gccnmf_klnmf_batched_workspace_bytes(B, F, T2, K))
        self.check(self.lib.gccnmf_klnmf_batched(self.h, V.data_ptr() if V.numel() else None, V.stride(1), V.stride(0), B, F, T2, _ptr(W), _ptr(H), K,
                                                 int(iterations), float(sparsity_alpha), float(epsilon), 1 if update_W else 0, _ptr(ws),
                                                 ws.numel(), self.stream))
        return W, H

    def klnmf_ragged(self, Vs, W, Hs, iterations, sparsity_alpha=0.0, epsilon=1e-16, update_W=True):
        """B clips of different lengths in one call, in place on W (B, F, K) and Hs[b] (K, T2_b) f32 cuda.  Vs[b] (F, T2_b) f32 cuda may be
        a strided view (unit stride along T2), e.g. a column range of one STFT output, read in place.  Clip b ends bit-identical to klnmf on
        it alone."""
        B = len(Vs)
        if B < 1 or len(Hs) != B:
            raise ParameterError('klnmf_ragged: %d V clips and %d H clips' % (B, len(Hs)))
        F, K = W.shape[1], W.shape[2]
        for b, (V, H) in enumerate(zip(Vs, Hs)):
            if not V.is_cuda or V.dim() != 2 or V.stride(1) != 1 or V.shape[0] != F:
                raise ParameterError('klnmf_ragged: V[%d] must be an (F, T2) cuda tensor with unit stride along T2' % b)
            if tuple(H.shape) != (K, V.shape[1]) or not H.is_contiguous():
                raise ParameterError('klnmf_ragged: H[%d] %s does not match V[%d] %s' % (b, tuple(H.shape), b, tuple(V.shape)))
        if tuple(W.shape) != (B, F, K) or not W.is_contiguous():
            raise ParameterError('klnmf_ragged: W %s is not a contiguous (%d, %d, %d) stack' % (tuple(W.shape), B, F, K))
        T2 = (c_int * B)(*[int(V.shape[1]) for V in Vs])
        Vp = (ctypes.c_void_p * B)(*[V.data_ptr() for V in Vs])
        ld = (c_int64 * B)(*[V.stride(0) for V in Vs])
        Hp = (ctypes.c_void_p * B)(*[H.data_ptr() for H in Hs])
        ws = self.workspace('klnmf_ragged', self.lib.gccnmf_klnmf_ragged_workspace_bytes(B, F, T2, K))
        self.check(self.lib.gccnmf_klnmf_ragged(self.h, Vp, ld, T2, B, F, _ptr(W), Hp, K, int(iterations), float(sparsity_alpha), float(epsilon),
                                                1 if update_W else 0, _ptr(ws), ws.numel(), self.stream))
        return W, Hs

    def _klnmf_ws(self, F, T2, K):
        return self.workspace('klnmf', self.lib.gccnmf_klnmf_workspace_bytes(F, T2, K))

    def klnmf_begin(self, V, W, H):
        F, T2 = V.shape
        K = W.shape[1]
        ws = self._klnmf_ws(F, T2, K)
        self.check(self.lib.gccnmf_klnmf_begin(self.h, _ptr(V), F, T2, _ptr(W), _ptr(H), K, _ptr(ws), ws.numel(), self.stream))

    def klnmf_step_numer(self, V, W, H, iteration, numer, sparsity_alpha=0.0, epsilon=1e-16):
        F, T2 = V.shape
        K = W.shape[1]
        ws = self._klnmf_ws(F, T2, K)
        self.check(self.lib.gccnmf_klnmf_step_numer(self.h, _ptr(V), F, T2, _ptr(W), _ptr(H), K, float(sparsity_alpha),
                                                    float(epsilon), int(iteration), _ptr(numer), _ptr(ws), ws.numel(), self.stream))

    def klnmf_step_apply(self, W, H, numer):
        F, K = W.shape
        T2 = H.shape[1]
        ws = self._klnmf_ws(F, T2, K)
        self.check(self.lib.gccnmf_klnmf_step_apply(self.h, F, T2, _ptr(W), _ptr(H), K, _ptr(numer), _ptr(ws), ws.numel(), self.stream))

    def klnmf_step_apply_multimem(self, W, H, numer_multicast_ptr):
        """W update reading the cross-rank numerator sum through the NVSwitch multicast address (an int)."""
        F, K = W.shape
        T2 = H.shape[1]
        ws = self._klnmf_ws(F, T2, K)
        self.check(self.lib.gccnmf_klnmf_step_apply_multimem(self.h, F, T2, _ptr(W), _ptr(H), K, int(numer_multicast_ptr), _ptr(ws),
                                                             ws.numel(), self.stream))

    def klnmf_step_multimem(self, V, W, H, iteration, numer_local_ptr, numer_multicast_ptr, counter_local_ptr, counter_multicast_ptr,
                            arrivals_expected, sparsity_alpha=0.0, epsilon=1e-16):
        """One sharded iteration with the exchange fused into the kernels (see gccnmf_klnmf_step_multimem); pointers are ints."""
        F, T2 = V.shape
        K = W.shape[1]
        ws = self._klnmf_ws(F, T2, K)
        self.check(self.lib.gccnmf_klnmf_step_multimem(self.h, _ptr(V), F, T2, _ptr(W), _ptr(H), K, float(sparsity_alpha), float(epsilon),
                                                       int(iteration), int(numer_local_ptr), int(numer_multicast_ptr), int(counter_local_ptr),
                                                       int(counter_multicast_ptr), int(arrivals_expected) & 0xFFFFFFFF, _ptr(ws), ws.numel(), self.stream))

    def klnmf_step_multimem2(self, V, W, H, iteration, rank, world, numer_local_ptr, numer_multicast_ptr, reduced_local_ptr,
                             reduced_multicast_ptr, counters_local_ptr, counters_multicast_ptr, arrivals_expected, sparsity_alpha=0.0,
                             epsilon=1e-16):
        """One sharded iteration with the two-shot in-switch exchange (see gccnmf_klnmf_step_multimem2); pointers are ints."""
        F, T2 = V.shape
        K = W.shape[1]
        ws = self._klnmf_ws(F, T2, K)
        self.check(self.lib.gccnmf_klnmf_step_multimem2(self.h, _ptr(V), F, T2, _ptr(W), _ptr(H), K, float(sparsity_alpha), float(epsilon),
                                                        int(iteration), int(rank), int(world), int(numer_local_ptr), int(numer_multicast_ptr),
                                                        int(reduced_local_ptr), int(reduced_multicast_ptr), int(counters_local_ptr),
                                                        int(counters_multicast_ptr), int(arrivals_expected) & 0xFFFFFFFF, _ptr(ws), ws.numel(),
                                                        self.stream))

    def klnmf_step_pull(self, V, W, H, iteration, epoch, rank, world, bases, layout_T2, two_shot, direct, sparsity_alpha=0.0, epsilon=1e-16):
        """One sharded iteration with the pull exchange (see gccnmf_klnmf_step_pull); bases: ctypes array of world void pointers."""
        F, T2 = V.shape
        K = W.shape[1]
        ws = self._klnmf_ws(F, T2, K)
        self.check(self.lib.gccnmf_klnmf_step_pull(self.h, _ptr(V), F, T2, _ptr(W), _ptr(H), K, float(sparsity_alpha), float(epsilon), int(iteration),
                                                   int(epoch), int(rank), int(world), bases, int(layout_T2), int(two_shot), int(direct), _ptr(ws), ws.numel(),
                                                   self.stream))

    def klnmf_end(self, W, H, iterations_done):
        F, K = W.shape
        T2 = H.shape[1]
        ws = self._klnmf_ws(F, T2, K)
        self.check(self.lib.gccnmf_klnmf_end(self.h, F, T2, _ptr(W), _ptr(H), K, int(iterations_done), _ptr(ws), ws.numel(), self.stream))

    def phat_angspec(self, X, E=None, want_coherence=True, want_angular=True, want_mean=True, out_key=None):
        """X (2, F, T) c64 mixture spectrogram -- or an (F, T) c64 coherence used as is -- and
        E (F, D) c128 -> (coherence (F,T) c64, angular (D,T) f64, mean (D) f64)."""
        torch = self.torch
        is_coh = X.dim() == 2
        F, T = X.shape[-2:]
        D = E.shape[1] if E is not None else 0
        coh = self._out(out_key, 'coh', (F, T), torch.complex64) if want_coherence else None
        ang = self._out(out_key, 'ang', (D, T), torch.float64) if (want_angular and D) else None
        mean = self._out(out_key, 'mean', (D,), torch.float64) if (want_mean and D) else None
        ws = self.workspace('angspec', self.lib.gccnmf_phat_angspec_workspace_bytes(F, T, max(D, 1)))
        self.check(self.lib.gccnmf_phat_angspec(self.h, _ptr(X), F, T, 1 if is_coh else 0, _ptr(E), D, _ptr(coh), _ptr(ang), _ptr(mean),
                                                _ptr(ws), ws.numel(), self.stream))
        return coh, ang, mean

    def tdoa_gccnmf(self, coherence, E, W, want_values=False, want_argmax=True):
        """coherence (F,T) c64, E (F,D) c128, W (F,K) f32 -> (values (D,K,T) f32 | None, argmax (K,T) i32 | None)."""
        torch = self.torch
        F, T = coherence.shape
        D = E.shape[1]
        K = W.shape[1]
        values = self.empty((D, K, T), torch.float32) if want_values else None
        argmax = self.empty((K, T), torch.int32) if want_argmax else None
        self.check(self.lib.gccnmf_tdoa_gccnmf(self.h, _ptr(coherence), F, T, _ptr(E), D, _ptr(W), K, _ptr(values),
                                               _ptr(argmax), self.stream))
        return values, argmax

    def tdoa_argmax(self, coherence, E, W, out_key=None):
        """argmax over all TDOAs (K, T) int32: tensor-core GEMM + exact float64 refinement of near-ties
        (float64 kernel for shapes the fast path does not cover).  Returns (argmax, refined_count tensor)."""
        torch = self.torch
        F, T = coherence.shape
        D, K = E.shape[1], W.shape[1]
        argmax = self._out(out_key, 'argmax', (K, T), torch.int32)
        refined = self._out(out_key, 'refined', (1,), torch.int32)
        ws = self.workspace('tdoa_argmax', self.lib.gccnmf_tdoa_argmax_workspace_bytes(F, T, D, K))
        self.check(self.lib.gccnmf_tdoa_argmax(self.h, _ptr(coherence), F, T, _ptr(E), D, _ptr(W), K, _ptr(argmax), _ptr(refined),
                                               _ptr(ws), ws.numel(), self.stream))
        return argmax, refined

    def coeff_mask(self, gccnmfs):
        torch = self.torch
        S, K, T = gccnmfs.shape
        masks = self.empty((S, K, T), torch.float32)
        flag = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.check(self.lib.gccnmf_coeff_mask(self.h, _ptr(gccnmfs), S, K, T, _ptr(masks), _ptr(flag), self.stream))
        return masks, flag

    def argmax_mask(self, argmax, lut, out_key=None):
        torch = self.torch
        K, T = argmax.shape
        mask = self._out(out_key, 'mask', (K, T), torch.float32)
        self.check(self.lib.gccnmf_argmax_mask(self.h, _ptr(argmax), K, T, _ptr(lut), lut.numel(), _ptr(mask), self.stream))
        return mask

    def window_targets(self, angular, window, P, want_means=True, out_key=None):
        """angular (D, T) f64 -> (targets (T, P) i32, means (D, T) f64 | None, status (1) i32): each frame's P targets from the
        nanmean of its newest `window` frames (gccnmf_window_targets); status bit 0 when a frame held earlier targets."""
        torch = self.torch
        D, T = angular.shape
        means = self._out(out_key, 'window_means', (D, T), torch.float64) if want_means else None
        targets = self._out(out_key, 'frame_targets', (T, int(P)), torch.int32)
        status = self._out(out_key, 'window_status', (1,), torch.int32)
        status.zero_()
        self.check(self.lib.gccnmf_window_targets(self.h, _ptr(angular), D, T, int(window), int(P), _ptr(means), _ptr(targets), _ptr(status),
                                                  self.stream))
        return targets, means, status

    def target_gccnmf(self, coherence, E, W, targets, out_key=None):
        """coherence (F, T) c64, E (F, D) c128, W (F, K) f32, targets (T, P) i32 -> values (P, K, T) f32 at each frame's targets.
        Every target must be in [0, D): the kernel indexes E with them unchecked (gccnmf_target_gccnmf), as window_targets writes them."""
        torch = self.torch
        F, T = coherence.shape
        D, K, P = E.shape[1], W.shape[1], targets.shape[1]
        values = self._out(out_key, 'target_values', (P, K, T), torch.float32)
        self.check(self.lib.gccnmf_target_gccnmf(self.h, _ptr(coherence), F, T, _ptr(E), D, _ptr(W), K, _ptr(targets), P, _ptr(values),
                                                 self.stream))
        return values

    def argmax_mask_frames(self, argmax, tdoas, targets, window_seconds, out_key=None):
        """argmax (K, T) i32, tdoas (D) f64, targets (T) i32 -> mask (K, T) f32 = |tdoa[argmax] - tdoa[target of the frame]| < window."""
        torch = self.torch
        K, T = argmax.shape
        D = tdoas.numel()
        table = self.workspace('tdoa_table', D * D)
        mask = self._out(out_key, 'mask', (K, T), torch.float32)
        self.check(self.lib.gccnmf_argmax_mask_frames(self.h, _ptr(argmax), K, T, _ptr(tdoas), D, _ptr(targets), float(window_seconds), _ptr(table),
                                                      _ptr(mask), self.stream))
        return mask

    def online_targets(self, angular):
        """angular (D, T) f64 -> (accumulated max (D, T) f64, targets (T) i32)."""
        torch = self.torch
        D, T = angular.shape
        acc = self.empty((D, T), torch.float64)
        targets = self.empty((T,), torch.int32)
        self.check(self.lib.gccnmf_online_targets(self.h, _ptr(angular), D, T, _ptr(acc), _ptr(targets), self.stream))
        return acc, targets

    def atom_mask(self, argmax, targets=None, target_scalar=0.0, epsilon=1.0, mode=0, beta=1.0, noise_floor=0.0):
        torch = self.torch
        K, T = argmax.shape
        mask = self.empty((K, T), torch.float32)
        self.check(self.lib.gccnmf_atom_mask(self.h, _ptr(argmax), K, T, _ptr(targets), float(target_scalar), float(epsilon),
                                             int(mode), float(beta), float(noise_floor), _ptr(mask), self.stream))
        return mask

    def wiener_apply(self, mask, W, X, want_filter=False):
        """mask (K, T) f32, W (F, K) f32, X (2, F, T) c64 -> Y (2, F, T) c64 [, wiener (F, T) f32]."""
        torch = self.torch
        K, T = mask.shape
        F = W.shape[0]
        Y = self.empty((2, F, T), torch.complex64)
        wiener = self.empty((F, T), torch.float32) if want_filter else None
        ws = self.workspace('wiener', self.lib.gccnmf_wiener_apply_workspace_bytes(F))
        self.check(self.lib.gccnmf_wiener_apply(self.h, _ptr(mask), _ptr(W), _ptr(X), F, T, K, _ptr(Y), _ptr(wiener), _ptr(ws),
                                                ws.numel(), self.stream))
        return (Y, wiener) if want_filter else Y

    def wiener_apply_h(self, mask, W, H, X, want_filter=False):
        """mask (K, T), W (F, K), H (K, 2T) [channel-major columns], X (2, F, T) c64 -> Y (2, F, T) c64 [, wiener (2, F, T) f32]."""
        torch = self.torch
        K, T = mask.shape
        F = W.shape[0]
        Y = self.empty((2, F, T), torch.complex64)
        wiener = self.empty((2, F, T), torch.float32) if want_filter else None
        self.check(self.lib.gccnmf_wiener_apply_h(self.h, _ptr(mask), _ptr(W), _ptr(H), _ptr(X), F, T, K, _ptr(Y), _ptr(wiener), self.stream))
        return (Y, wiener) if want_filter else Y

    def masked_recon_phase(self, masks, X, W, H, out_key=None, tensor_cores=True):
        """masks (S,K,T) f32, X (2,F,T) c64, W (F,K), H (K,2T) -> (S,2,F,T) c64."""
        torch = self.torch
        S, K, T = masks.shape
        F = X.shape[1]
        out = self._out(out_key, 'est', (S, 2, F, T), torch.complex64)
        ws = self.workspace('masked_recon', self.lib.gccnmf_masked_recon_workspace_bytes(S, F, T, K)) if tensor_cores else None
        self.check(self.lib.gccnmf_masked_recon_phase(self.h, _ptr(masks), _ptr(X), _ptr(W), _ptr(H), S, F, T, K,
                                                      _ptr(out), _ptr(ws), ws.numel() if ws is not None else 0, self.stream))
        return out


    def gemm_planes(self, A, B, a_mn_major=False, b_mn_major=False, tile_n=128, splits=1, timing=None):
        """(A . B^T)^T on the TMA-fed plane GEMM.  A: (M, Kc) or, MN-major, (Kc, M); B likewise with N.
        Returns DT (splits, N, M) f32 (partial slabs over k ranges when splits > 1)."""
        torch = self.torch
        M, Kc = (A.shape[1], A.shape[0]) if a_mn_major else A.shape
        N = B.shape[1] if b_mn_major else B.shape[0]
        DT = self.empty((splits, N, M), torch.float32)
        ws = self.workspace('gemm_planes', self.lib.gccnmf_gemm_planes_workspace_bytes(M, N, Kc))
        self.check(self.lib.gccnmf_gemm_planes(self.h, _ptr(A), 1 if a_mn_major else 0, _ptr(B), 1 if b_mn_major else 0, _ptr(DT),
                                               M, N, Kc, tile_n, splits, _ptr(ws), ws.numel(), _ptr(timing), self.stream))
        return DT


_default_handles = {}


def default_handle(device=None):
    """Process-wide handle per device (created lazily; raises without a GPU).  device None: the reference's functions take no device
    argument -- $GCCNMF_DEVICE if set, else torch's current device (what a torchrun rank selected with torch.cuda.set_device)."""
    if device is None:
        env = os.environ.get('GCCNMF_DEVICE')
        if env is not None:
            device = int(env)
        else:
            import torch
            device = torch.cuda.current_device() if torch.cuda.is_available() else 0
    h = _default_handles.get(device)
    if h is None:
        h = _default_handles[device] = Handle(device)
    return h
