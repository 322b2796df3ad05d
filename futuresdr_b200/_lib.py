"""ctypes binding of libb200sdr.so (include/b200sdr.h).

The product path is the CUDA library and nothing else: if ``libb200sdr.so`` is missing or does
not export a symbol the header declares, importing this module raises -- there is no CPU
fallback anywhere under ``futuresdr_b200/``.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# B2S_LIB lets a developer A/B a differently-built library (kernel tuning); default is the in-tree build
SO_PATH = os.environ.get("B2S_LIB") or os.path.join(_HERE, "libb200sdr.so")

OK, EINVAL, ECUDA, ENOMEM, EAGAIN, EUNSUPPORTED, ESTATE, ETIMEOUT = 0, -1, -2, -3, -4, -5, -6, -7
INSUFFICIENT_INPUT, INSUFFICIENT_OUTPUT, BOTH_SUFFICIENT = 0, 1, 2
F32_F32, C32_F32, C32_C32, F64_F64 = 0, 1, 2, 3
ALGO_AUTO, ALGO_DIRECT, ALGO_TENSOR, ALGO_FFT, ALGO_SCAN = 0, 1, 2, 3, 4
(OP_SCALE_F32, OP_SCALE_C32, OP_QUAD_DEMOD, OP_NORM_SQR, OP_QUAD_DEMOD_C32, OP_EXP_F32,
 OP_MAG_C32, OP_LOG10_F32, OP_DC_BLOCK_F32, OP_SLICE_F32_U8, OP_DIV_C32, OP_C32_TO_I16_IQ) = range(12)
MIX_ROTATE_C32, MIX_ROTATE_SCALE_C32, MIX_WEAVER_F32 = 0, 1, 2
KEYFOB_NONE, KEYFOB_CLOSE, KEYFOB_OPEN, KEYFOB_TRUNK = 0, 1, 2, 3
WAVE_COS, WAVE_SIN, WAVE_SQUARE = 0, 1, 2
(COMBINE_ADD_F32, COMBINE_SUB_F32, COMBINE_MUL_F32, COMBINE_CONJ_MUL_C32, COMBINE_MAG_DIV_C32_F32, COMBINE_TO_C32,
 COMBINE_TO_C32_NEG_Q) = range(7)
SPLIT_RE_IM, SPLIT_DUP_F32 = 0, 1
FANOUT_MAX_OUTPUTS = 256
LORA_MAX_PAYLOAD = 255
WLAN_MAX_PAYLOAD = 1500
WLAN_MAX_PSDU = 1528
ZIGBEE_MAX_PAYLOAD = 116
ZIGBEE_PADDING = 40000

_vp, _sz, _i32, _f32 = C.c_void_p, C.c_size_t, C.c_int32, C.c_float
_szp, _i32p, _vpp, _f32p = C.POINTER(C.c_size_t), C.POINTER(C.c_int32), C.POINTER(C.c_void_p), C.POINTER(C.c_float)

# name -> (restype, argtypes): one entry per function declared in include/b200sdr.h
SIGNATURES = {
    "b2s_version": (_i32, []),
    "b2s_ctx_create": (_i32, [C.c_int, _vpp]),
    "b2s_ctx_create_on_stream": (_i32, [C.c_int, _vp, _vpp]),
    "b2s_ctx_destroy": (None, [_vp]),
    "b2s_last_error": (C.c_char_p, [_vp]),
    "b2s_ctx_sync": (_i32, [_vp]),
    "b2s_ctx_stream": (_vp, [_vp]),
    "b2s_ctx_sm_count": (_i32, [_vp]),
    "b2s_ctx_launch_count": (C.c_uint64, [_vp]),
    "b2s_ctx_bytes_held": (C.c_uint64, [_vp]),
    "b2s_malloc": (_i32, [_vp, _sz, _vpp]),
    "b2s_free": (_i32, [_vp, _vp]),
    "b2s_host_alloc": (_i32, [_vp, _sz, _vpp]),
    "b2s_host_free": (_i32, [_vp, _vp]),
    "b2s_memcpy_h2d": (_i32, [_vp, _vp, _vp, _sz]),
    "b2s_memcpy_d2h": (_i32, [_vp, _vp, _vp, _sz]),
    "b2s_fir_plan": (_i32, [_vp, C.c_int, _f32p, _sz, _sz, _vpp]),
    "b2s_fir_plan_f32_f32": (_i32, [_vp, _f32p, _sz, _sz, _vpp]),
    "b2s_fir_plan_c32_f32": (_i32, [_vp, _f32p, _sz, _sz, _vpp]),
    "b2s_fir_plan_c32_c32": (_i32, [_vp, _f32p, _sz, _sz, _vpp]),
    "b2s_fir_plan_f64_f64": (_i32, [_vp, C.POINTER(C.c_double), _sz, _sz, _vpp]),
    "b2s_fir_destroy": (None, [_vp]),
    "b2s_fir_length": (_sz, [_vp]),
    "b2s_fir_set_algo": (_i32, [_vp, C.c_int]),
    "b2s_fir_get_algo": (_i32, [_vp]),
    "b2s_fir_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp, _i32p]),
    "b2s_fir_filter_host": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp, _i32p]),
    "b2s_fir_exec_hist": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp, _szp, _szp, _i32p]),
    "b2s_resamp_plan": (_i32, [_vp, C.c_int, _f32p, _sz, _sz, _sz, _vpp]),
    "b2s_resamp_destroy": (None, [_vp]),
    "b2s_resamp_length": (_sz, [_vp]),
    "b2s_resamp_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp, _i32p]),
    "b2s_pfbarb_plan_c32": (_i32, [_vp, _f32p, _sz, _sz, _f32, _vpp]),
    "b2s_pfbarb_destroy": (None, [_vp]),
    "b2s_pfbarb_reset": (_i32, [_vp]),
    "b2s_pfbarb_period": (_i32, [_f32, _sz, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "b2s_pfbarb_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp, _i32p]),
    "b2s_fft_plan_c32": (_i32, [_vp, _sz, _i32, _i32, _i32, _f32, _vpp]),
    "b2s_fft_destroy": (None, [_vp]),
    "b2s_fft_length": (_sz, [_vp]),
    "b2s_fft_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp]),
    "b2s_apply_create": (_i32, [_vp, C.c_int, _f32, _vpp]),
    "b2s_apply_destroy": (None, [_vp]),
    "b2s_apply_reset": (_i32, [_vp]),
    "b2s_apply_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp]),
    "b2s_rotator_create": (_i32, [_vp, _f32, _vpp]),
    "b2s_rotator_destroy": (None, [_vp]),
    "b2s_rotator_reset": (_i32, [_vp]),
    "b2s_rotator_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _i32p]),
    "b2s_xlating_taps": (_i32, [_f32p, _sz, _f32, _f32, _sz, _f32p, _f32p]),
    "b2s_mixer_create": (_i32, [_vp, C.c_int, _f32, _f32, _vpp]),
    "b2s_mixer_destroy": (None, [_vp]),
    "b2s_mixer_reset": (_i32, [_vp]),
    "b2s_mixer_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp]),
    "b2s_chan_plan_c32": (_i32, [_vp, _sz, _f32p, _sz, _f32, _vpp]),
    "b2s_chan_destroy": (None, [_vp]),
    "b2s_chan_decimation": (_sz, [_vp]),
    "b2s_chan_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _sz, _szp, _szp, _i32p]),
    "b2s_synth_plan_c32": (_i32, [_vp, _sz, _f32p, _sz, _vpp]),
    "b2s_synth_destroy": (None, [_vp]),
    "b2s_synth_exec": (_i32, [_vp, _vp, _sz, _sz, _vp, _sz, _szp, _szp]),
    "b2s_mavg_create": (_i32, [_vp, _sz, _f32, _sz, _vpp]),
    "b2s_mavg_destroy": (None, [_vp]),
    "b2s_mavg_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp]),
    "b2s_iir_plan_f32": (_i32, [_vp, _f32p, _sz, _f32p, _sz, _vpp]),
    "b2s_iir_plan_f64": (_i32, [_vp, C.POINTER(C.c_double), _sz, C.POINTER(C.c_double), _sz, _vpp]),
    "b2s_iir_destroy": (None, [_vp]),
    "b2s_iir_length": (_sz, [_vp]),
    "b2s_iir_set_algo": (_i32, [_vp, C.c_int]),
    "b2s_iir_get_algo": (_i32, [_vp]),
    "b2s_iir_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp, _i32p]),
    "b2s_sigsrc_create": (_i32, [_vp, C.c_int, _i32, _f32, _f32, _f32, _f32, _vpp]),
    "b2s_sigsrc_destroy": (None, [_vp]),
    "b2s_sigsrc_set_amplitude": (_i32, [_vp, _f32]),
    "b2s_sigsrc_phase": (_i32, [_vp, _i32p, _i32p]),
    "b2s_sigsrc_exec": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_fxpt_phase_new": (_i32, [_f32, _i32p]),
    "b2s_fxpt_sin_cos": (_i32, [_i32, _f32p, _f32p]),
    "b2s_spectrum_plan":(_i32, [_vp, _sz, _i32, _f32, _sz, _f32, _vpp]),
    "b2s_spectrum_destroy": (None, [_vp]),
    "b2s_spectrum_reset": (_i32, [_vp]),
    "b2s_spectrum_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp]),
    "b2s_ring_create": (_i32, [_vp, _sz, _sz, _sz, _i32, _i32, _vpp]),
    "b2s_ring_destroy": (None, [_vp]),
    "b2s_ring_acquire_empty": (_i32, [_vp, _vpp]),
    "b2s_ring_submit_full": (_i32, [_vp, _vp, _sz, _i32]),
    "b2s_ring_acquire_full": (_i32, [_vp, _vpp, _szp]),
    "b2s_ring_release": (_i32, [_vp, _vp]),
    "b2s_ring_carry_halo": (_i32, [_vp, _vp, _sz, _sz, _vp]),
    "b2s_slot_device_ptr": (_vp, [_vp]),
    "b2s_slot_host_ptr": (_vp, [_vp]),
    "b2s_slot_halo_valid": (_sz, [_vp]),
    "b2s_slot_fetch_to_host": (_i32, [_vp, _sz]),
    "b2s_slot_wait": (_i32, [_vp]),
    "b2s_ring_free_slots": (_sz, [_vp]),
    "b2s_ring_full_slots": (_sz, [_vp]),
    "b2s_ring_base": (_vp, [_vp]),
    "b2s_ring_bytes": (_sz, [_vp]),
    "b2s_ring_slot_offset": (_sz, [_vp, _i32]),
    "b2s_ring_flags_offset": (_sz, [_vp]),
    "b2s_slot_index": (_i32, [_vp]),
    "b2s_ipc_export": (_i32, [_vp, _vp, _vp]),
    "b2s_ipc_open": (_i32, [_vp, _vp, _vpp]),
    "b2s_ipc_close": (_i32, [_vp, _vp]),
    "b2s_peer_enable": (_i32, [_vp, _i32]),
    "b2s_flag_set": (_i32, [_vp, _vp, C.c_uint32]),
    "b2s_flag_wait": (_i32, [_vp, _vp, C.c_uint32]),
    "b2s_flag_read": (_i32, [_vp, _vp, C.POINTER(C.c_uint32)]),
    "b2s_memcpy_d2d": (_i32, [_vp, _vp, _vp, _sz]),
    "b2s_memset": (_i32, [_vp, _vp, _i32, _sz]),
    "b2s_firdes_kaiser_lowpass": (_sz, [C.c_double, C.c_double, C.c_double, _f32p, _sz]),
    "b2s_firdes_kaiser_multirate": (_sz, [_sz, _sz, _sz, C.c_double, _f32p, _sz]),
    "b2s_combine_exec": (_i32, [_vp, C.c_int, _vp, _sz, _vp, _sz, _vp, _sz, _szp, _szp]),
    "b2s_split_exec": (_i32, [_vp, C.c_int, _vp, _sz, _vp, _vp, _sz, _szp, _szp]),
    "b2s_fanout_exec": (_i32, [_vp, _i32, _sz, _vp, _sz, _vpp, _sz, _sz, _szp, _szp]),
    "b2s_boxavg_create": (_i32, [_vp, _i32, _sz, _i32, _f32, _vpp]),
    "b2s_boxavg_destroy": (None, [_vp]),
    "b2s_boxavg_reset": (_i32, [_vp]),
    "b2s_boxavg_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _sz, _szp, _szp, _szp, _i32p, _i32p]),
    "b2s_adsb_create": (_i32, [_vp, _f32, _i32, _vpp]),
    "b2s_adsb_destroy": (None, [_vp]),
    "b2s_adsb_reset": (_i32, [_vp]),
    "b2s_adsb_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _i32, _szp, _i32p]),
    "b2s_adsb_drain_packets": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_adsb_drain_detections": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_mmclock_create": (_i32, [_vp, _f32, _f32, _f32, _f32, _f32, _vpp]),
    "b2s_mmclock_destroy": (None, [_vp]),
    "b2s_mmclock_reset": (_i32, [_vp]),
    "b2s_mmclock_look_ahead": (_sz, [_vp]),
    "b2s_mmclock_exec": (_i32, [_vp, _vp, _sz, _vp, _sz, _szp, _szp]),
    "b2s_zigbee_create": (_i32, [_vp, C.c_uint32, _vpp]),
    "b2s_zigbee_destroy": (None, [_vp]),
    "b2s_zigbee_reset": (_i32, [_vp]),
    "b2s_zigbee_exec": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_zigbee_drain_frames": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_window_hamming": (_sz, [_sz, _i32, C.POINTER(C.c_double), _sz]),
    "b2s_firdes_hilbert": (_sz, [C.POINTER(C.c_double), _sz, _f32p, _sz]),
    "b2s_keyfob_create": (_i32, [_vp, _vpp]),
    "b2s_keyfob_destroy": (None, [_vp]),
    "b2s_keyfob_reset": (_i32, [_vp]),
    "b2s_keyfob_exec": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_keyfob_drain_codes": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_firdes_lowpass": (_sz, [C.c_double, C.POINTER(C.c_double), _sz, _f32p, _sz]),
    "b2s_lora_symbol_count": (_i32, [_i32, _i32, _i32, _i32, _i32, _sz, _szp]),
    "b2s_lora_encode": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _vp, _szp, _sz, _vp, _sz, _szp]),
    "b2s_lora_tx_create": (_i32, [_vp, _i32, _i32, _i32, _i32, _i32, _sz, C.POINTER(C.c_uint32), _sz, _sz, _vpp]),
    "b2s_lora_tx_destroy": (None, [_vp]),
    "b2s_lora_tx_reset": (_i32, [_vp]),
    "b2s_lora_tx_push": (_i32, [_vp, _vp, _szp, _sz]),
    "b2s_lora_tx_set_sync_word": (_i32, [_vp, C.c_uint32, C.c_uint32]),
    "b2s_lora_tx_finish": (_i32, [_vp]),
    "b2s_lora_tx_pending": (_i32, [_vp, C.POINTER(C.c_uint64)]),
    "b2s_lora_tx_exec": (_i32, [_vp, _vp, _sz, _szp, _i32p]),
    "b2s_lora_tx_drain_bursts": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_wlan_frame_param": (_i32, [_i32, _sz, _szp, _szp, _szp]),
    "b2s_wlan_encode": (_i32, [_vp, _vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp, _szp, _i32p, _sz, _vp, _sz, _szp]),
    "b2s_wlan_tx_create": (_i32, [_vp, _vp, _vp, _vp, _i32, _sz, _sz, _vpp]),
    "b2s_wlan_tx_destroy": (None, [_vp]),
    "b2s_wlan_tx_reset": (_i32, [_vp]),
    "b2s_wlan_tx_push": (_i32, [_vp, _vp, _szp, _i32p, _sz]),
    "b2s_wlan_tx_finish": (_i32, [_vp]),
    "b2s_wlan_tx_pending": (_i32, [_vp, C.POINTER(C.c_uint64)]),
    "b2s_wlan_tx_exec": (_i32, [_vp, _vp, _sz, _szp, _i32p]),
    "b2s_wlan_tx_drain_bursts": (_i32, [_vp, _vp, _sz, _szp]),
    "b2s_zigbee_tx_create": (_i32, [_vp, _sz, _vpp]),
    "b2s_zigbee_tx_destroy": (None, [_vp]),
    "b2s_zigbee_tx_reset": (_i32, [_vp]),
    "b2s_zigbee_tx_push": (_i32, [_vp, _vp, _szp, _sz, _szp]),
    "b2s_zigbee_tx_finish": (_i32, [_vp]),
    "b2s_zigbee_tx_pending": (_i32, [_vp, C.POINTER(C.c_uint64)]),
    "b2s_zigbee_tx_exec": (_i32, [_vp, _vp, _sz, _szp, _i32p]),
    "b2s_zigbee_tx_drain_bursts": (_i32, [_vp, _vp, _sz, _szp]),
}


class Handshake(C.Structure):
    """b2s_handshake (include/b200sdr.h): the cross-GPU flags of one b2s_fir_exec_hist call."""
    _fields_ = [("publish_flag", C.c_void_p), ("publish_value", C.c_uint32),
                ("wait_flag", C.c_void_p), ("wait_value", C.c_uint32),
                ("done_flag", C.c_void_p), ("done_value", C.c_uint32)]


class B200SdrError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libb200sdr error {code}: {msg}")
        self.code = code


def _load() -> C.CDLL:
    if not os.path.exists(SO_PATH):
        raise ImportError(
            f"{SO_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C futuresdr_b200/csrc`). futuresdr_b200 has no CPU fallback."
        )
    lib = C.CDLL(SO_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise ImportError(f"{SO_PATH} does not export {name} (stale build?)") from e
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


class Handle:
    """Owner of one C-ABI handle ``self._h``: ``close()`` -- and, failing that, ``__del__`` -- passes it to the class's
    ``_destroy`` exactly once."""
    _destroy = None

    def close(self):
        if getattr(self, "_h", None):
            type(self)._destroy(self._h)
            self._h = None

    def __del__(self):
        try:                                   # (module globals may already be gone at interpreter shutdown)
            self.close()
        except Exception:  # noqa: BLE001
            pass


def check(rc: int, ctx=None):
    if rc < 0:
        msg = lib.b2s_last_error(ctx)
        raise B200SdrError(rc, msg.decode() if msg else "")
    return rc
