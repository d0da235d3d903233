"""ctypes binding of include/fsk_b200.h.

Mirrors the reference's operator interface for the hot path:

* :class:`FskPlan` -- ``fsk_plan_new`` / ``fsk_find_frame`` / ``fsk_detect_carrier`` /
  ``fsk_set_tones_by_bandshift`` / ``fsk_plan_destroy`` with the reference's
  argument meaning (src/fsk.h:49-78), host sample buffers;
* :class:`RxEngine` -- the batched extension: ``find_frame_batch`` (one
  src/fsk.c:449 search per stream) and ``rx_batch`` (the whole rx loop,
  src/minimodem.c:1137-1463, per stream) on device-resident torch tensors,
  ``rx_batch_host`` on host arrays.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FSK_B200_LIB") or os.path.join(_HERE, "libfsk_b200.so")   # override: tuning builds
MAX_BITS = 64
FRAME_ACQUIRED = 0x80000000
FRAME_REPORT = 0xFFFFFFFF


class RxConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_float), ("data_rate", C.c_float),
                ("f_mark", C.c_float), ("f_space", C.c_float), ("inverted", C.c_int),
                ("band_width", C.c_float), ("n_data_bits", C.c_uint), ("nstartbits", C.c_int),
                ("nstopbits", C.c_float), ("invert_start_stop", C.c_int), ("msb_first", C.c_int),
                ("do_rx_sync", C.c_int), ("sync_byte", C.c_ulonglong),
                ("confidence_threshold", C.c_float), ("confidence_search_limit", C.c_float),
                ("expect_data_string", C.c_char * (MAX_BITS + 4))]


class RxParams(C.Structure):
    _fields_ = [("sample_rate", C.c_float), ("f_mark", C.c_float), ("f_space", C.c_float),
                ("band_width", C.c_float), ("fftsize", C.c_int), ("nbands", C.c_uint),
                ("b_mark", C.c_uint), ("b_space", C.c_uint),
                ("nsamples_per_bit", C.c_float), ("frame_n_bits", C.c_uint),
                ("frame_nsamples", C.c_uint), ("expect_n_bits", C.c_uint),
                ("expect_nsamples", C.c_uint), ("nsamples_overscan", C.c_uint),
                ("try_max_nocarrier", C.c_uint), ("try_max_carrier", C.c_uint),
                ("confidence_threshold", C.c_float), ("confidence_search_limit", C.c_float),
                ("n_data_bits", C.c_uint), ("nstartbits", C.c_int), ("nstopbits", C.c_float),
                ("msb_first", C.c_int), ("do_rx_sync", C.c_int), ("sync_byte", C.c_ulonglong),
                ("samples_per_bit", C.c_float), ("bit_nsamples", C.c_uint),
                ("bit_begin", C.c_uint * MAX_BITS), ("span_nsamples", C.c_uint),
                ("expect_data", C.c_char * (MAX_BITS + 4)), ("expect_sync", C.c_char * (MAX_BITS + 4))]


class Frame(C.Structure):
    _fields_ = [("bits_lo", C.c_uint32), ("bits_hi", C.c_uint32), ("confidence", C.c_float),
                ("amplitude", C.c_float), ("frame_start", C.c_uint32)]


FRAME_DTYPE = np.dtype([("bits_lo", "<u4"), ("bits_hi", "<u4"), ("confidence", "<f4"),
                        ("amplitude", "<f4"), ("frame_start", "<u4")])


class StreamState(C.Structure):
    _fields_ = [("pos", C.c_uint64), ("nframes", C.c_uint32), ("carrier", C.c_uint32),
                ("noconfidence", C.c_uint32), ("track_amplitude", C.c_float),
                ("peak_confidence", C.c_float), ("done", C.c_uint32),
                ("carrier_nsamples", C.c_uint64), ("confidence_total", C.c_float),
                ("amplitude_total", C.c_float), ("nframes_decoded", C.c_uint32),
                ("stat_candidates", C.c_uint32), ("stat_searches", C.c_uint32), ("reserved", C.c_uint32)]


STATE_DTYPE = np.dtype([("pos", "<u8"), ("nframes", "<u4"), ("carrier", "<u4"),
                        ("noconfidence", "<u4"), ("track_amplitude", "<f4"),
                        ("peak_confidence", "<f4"), ("done", "<u4"),
                        ("carrier_nsamples", "<u8"), ("confidence_total", "<f4"),
                        ("amplitude_total", "<f4"), ("nframes_decoded", "<u4"),
                        ("stat_candidates", "<u4"), ("stat_searches", "<u4"), ("reserved", "<u4")])
STATE_WORDS = STATE_DTYPE.itemsize // 4


class TxConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_float), ("data_rate", C.c_float), ("f_mark", C.c_float),
                ("f_space", C.c_float), ("n_data_bits", C.c_uint), ("nstartbits", C.c_float),
                ("nstopbits", C.c_float), ("invert_start_stop", C.c_int), ("msb_first", C.c_int),
                ("do_tx_sync_bytes", C.c_uint), ("sync_byte", C.c_uint),
                ("leader_bits", C.c_int), ("trailer_bits", C.c_int)]


class TxSignal(C.Structure):
    """fsk_b200_tx_signal: --volume, --lut, --float-samples."""
    _fields_ = [("amplitude", C.c_float), ("sin_table_len", C.c_uint32), ("float_samples", C.c_int)]


class TxState(C.Structure):
    """fsk_b200_tx_state, 16 bytes per stream; all zeros = a fresh reference process."""
    _fields_ = [("cphase", C.c_float), ("baudot_charset", C.c_uint32), ("transmitting", C.c_uint32),
                ("reserved", C.c_uint32)]


TX_STATE_BYTES = 16
TX_IDLE_IF_EMPTY, TX_FINAL = 1, 2
ENCODE_ASCII8, ENCODE_BAUDOT = 0, 1


class FskPlanStruct(C.Structure):
    """struct fsk_plan, include/fsk_b200.h (layout of src/fsk.h:30-46)."""
    _fields_ = [("sample_rate", C.c_float), ("f_mark", C.c_float), ("f_space", C.c_float),
                ("filter_bw", C.c_float), ("fftsize", C.c_int), ("nbands", C.c_uint),
                ("band_width", C.c_float), ("b_mark", C.c_uint), ("b_space", C.c_uint),
                ("engine", C.c_void_p), ("scratch_in", C.c_void_p), ("scratch_out", C.c_void_p)]


EXPORTS = [
    "fsk_plan_new", "fsk_plan_destroy", "fsk_find_frame", "fsk_detect_carrier",
    "fsk_set_tones_by_bandshift",
    "fsk_b200_rx_config_for_mode", "fsk_b200_rx_params_derive", "fsk_b200_engine_new",
    "fsk_b200_engine_destroy", "fsk_b200_engine_params", "fsk_b200_engine_tune",
    "fsk_b200_find_frame_batch", "fsk_b200_find_frame_batch_bits", "fsk_b200_rx_batch", "fsk_b200_rx_batch_s16", "fsk_b200_rx_batch_host",
    "fsk_b200_max_frames", "fsk_b200_frame_databits", "fsk_b200_tx_batch", "fsk_b200_sin_table",
    "fsk_b200_s16_to_f32", "fsk_b200_rx_batch_host_s16", "fsk_b200_decode_ascii_batch",
    "fsk_b200_decode_batch", "fsk_b200_decoder_for_mode", "fsk_b200_decode_max_bytes_per_frame",
    "fsk_b200_decode_max_bytes", "fsk_b200_detect_carrier_batch",
    "fsk_b200_stream_window", "fsk_b200_engine_set_holdback", "fsk_b200_stream_push", "fsk_b200_wav_locate",
    "fsk_b200_version", "fsk_b200_launch_count", "fsk_b200_last_error", "fsk_b200_engine_last_kernel",
    "fsk_b200_encoder_for_mode", "fsk_b200_tx_config_from_rx", "fsk_b200_tx_engine_new", "fsk_b200_tx_engine_destroy",
    "fsk_b200_tx_max_samples", "fsk_b200_tx_text_batch",
]

_lib = None
# set by tests/emu/emu_mode.py only: lets the parity tests run against the host emulation build
ALLOW_NON_PRODUCT_LIBRARY = False


def build(force=False):
    """Compile libfsk_b200.so in-tree (nvcc, sm_90a; gcc for the host layer)."""
    args = ["make", "-s", "-C", os.path.join(_HERE, "csrc")]
    if force:
        subprocess.check_call(args + ["clean"])
    subprocess.check_call(args)
    return LIB_PATH


def lib():
    """Load the C-ABI library.  Fails loudly when it is missing: there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("%s is missing: build it with minimodem_b200.build() "
                           "(make -C minimodem_b200/csrc); there is no CPU/PyTorch fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.fsk_b200_version.restype = C.c_char_p
    if b"sm_90a" not in L.fsk_b200_version() and not ALLOW_NON_PRODUCT_LIBRARY:
        # FSK_B200_LIB exists for tuning builds of the CUDA library; anything else (the tests' host
        # emulation of the kernels, tests/emu) must never stand in for it silently
        raise RuntimeError("%s is not a build of the sm_90a library (%s); the binding refuses it"
                           % (LIB_PATH, L.fsk_b200_version().decode()))
    fp, u32p = C.POINTER(C.c_float), C.c_void_p
    L.fsk_plan_new.argtypes = [C.c_float] * 4
    L.fsk_plan_new.restype = C.POINTER(FskPlanStruct)
    L.fsk_plan_destroy.argtypes = [C.POINTER(FskPlanStruct)]
    L.fsk_plan_destroy.restype = None
    L.fsk_find_frame.argtypes = [C.POINTER(FskPlanStruct), fp, C.c_uint, C.c_uint, C.c_uint, C.c_uint,
                                 C.c_float, C.c_char_p, C.POINTER(C.c_ulonglong), fp, C.POINTER(C.c_uint)]
    L.fsk_find_frame.restype = C.c_float
    L.fsk_detect_carrier.argtypes = [C.POINTER(FskPlanStruct), fp, C.c_uint, C.c_float]
    L.fsk_detect_carrier.restype = C.c_int
    L.fsk_set_tones_by_bandshift.argtypes = [C.POINTER(FskPlanStruct), C.c_uint, C.c_int]
    L.fsk_set_tones_by_bandshift.restype = None
    L.fsk_b200_rx_config_for_mode.argtypes = [C.c_char_p, C.c_float, C.POINTER(RxConfig), C.POINTER(RxConfig)]
    L.fsk_b200_rx_config_for_mode.restype = C.c_int
    L.fsk_b200_rx_params_derive.argtypes = [C.POINTER(RxConfig), C.POINTER(RxParams)]
    L.fsk_b200_rx_params_derive.restype = C.c_int
    L.fsk_b200_engine_new.argtypes = [C.POINTER(RxParams)]
    L.fsk_b200_engine_new.restype = C.c_void_p
    L.fsk_b200_engine_destroy.argtypes = [C.c_void_p]
    L.fsk_b200_engine_destroy.restype = None
    L.fsk_b200_engine_params.argtypes = [C.c_void_p]
    L.fsk_b200_engine_params.restype = C.POINTER(RxParams)
    L.fsk_b200_engine_last_kernel.argtypes = [C.c_void_p]
    L.fsk_b200_engine_last_kernel.restype = C.c_char_p
    L.fsk_b200_engine_tune.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.fsk_b200_engine_tune.restype = C.c_int
    L.fsk_b200_find_frame_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, u32p, u32p,
                                            u32p, u32p, u32p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fsk_b200_find_frame_batch.restype = C.c_int
    L.fsk_b200_find_frame_batch_bits.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, u32p, u32p,
                                                 u32p, u32p, u32p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_void_p]
    L.fsk_b200_find_frame_batch_bits.restype = C.c_int
    L.fsk_b200_rx_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, u32p, C.c_uint32,
                                    C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.fsk_b200_rx_batch.restype = C.c_int
    L.fsk_b200_rx_batch_s16.argtypes = L.fsk_b200_rx_batch.argtypes
    L.fsk_b200_rx_batch_s16.restype = C.c_int
    L.fsk_b200_rx_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_uint32,
                                         C.c_void_p, C.c_uint32, C.c_void_p]
    L.fsk_b200_rx_batch_host.restype = C.c_int
    L.fsk_b200_max_frames.argtypes = [C.POINTER(RxParams), C.c_uint32]
    L.fsk_b200_max_frames.restype = C.c_uint32
    L.fsk_b200_frame_databits.argtypes = [C.POINTER(RxParams), C.POINTER(Frame)]
    L.fsk_b200_frame_databits.restype = C.c_ulonglong
    L.fsk_b200_tx_batch.argtypes = [C.POINTER(TxConfig), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                    C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_uint32, C.c_void_p]
    L.fsk_b200_tx_batch.restype = C.c_int
    L.fsk_b200_s16_to_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]
    L.fsk_b200_s16_to_f32.restype = C.c_int
    L.fsk_b200_rx_batch_host_s16.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_uint32,
                                             C.c_void_p, C.c_uint32, C.c_void_p]
    L.fsk_b200_rx_batch_host_s16.restype = C.c_int
    L.fsk_b200_decode_ascii_batch.argtypes = [C.POINTER(RxParams), C.c_void_p, C.c_void_p, C.c_size_t,
                                              C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.fsk_b200_decode_ascii_batch.restype = C.c_int
    L.fsk_b200_decode_batch.argtypes = [C.POINTER(RxParams), C.c_int, C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                        C.c_void_p]
    L.fsk_b200_decode_batch.restype = C.c_int
    L.fsk_b200_decoder_for_mode.argtypes = [C.c_char_p, C.c_uint, C.c_int]
    L.fsk_b200_decoder_for_mode.restype = C.c_int
    L.fsk_b200_decode_max_bytes_per_frame.argtypes = [C.c_int, C.c_uint]
    L.fsk_b200_decode_max_bytes_per_frame.restype = C.c_uint32
    L.fsk_b200_decode_max_bytes.argtypes = [C.c_int, C.c_uint, C.c_uint32]
    L.fsk_b200_decode_max_bytes.restype = C.c_uint64
    L.fsk_b200_detect_carrier_batch.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p,
                                                C.c_uint32, C.c_float, C.c_void_p, C.c_void_p]
    L.fsk_b200_detect_carrier_batch.restype = C.c_int
    L.fsk_b200_stream_window.argtypes = [C.POINTER(RxParams)]
    L.fsk_b200_stream_window.restype = C.c_uint32
    L.fsk_b200_engine_set_holdback.argtypes = [C.c_void_p, C.c_uint32]
    L.fsk_b200_engine_set_holdback.restype = C.c_int
    L.fsk_b200_stream_push.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.fsk_b200_stream_push.restype = C.c_int
    L.fsk_b200_wav_locate.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t),
                                      C.POINTER(C.c_uint32), C.POINTER(C.c_int)]
    L.fsk_b200_wav_locate.restype = C.c_int
    L.fsk_b200_encoder_for_mode.argtypes = [C.c_char_p, C.c_uint]
    L.fsk_b200_encoder_for_mode.restype = C.c_int
    L.fsk_b200_tx_config_from_rx.argtypes = [C.POINTER(RxConfig), C.POINTER(TxConfig)]
    L.fsk_b200_tx_config_from_rx.restype = C.c_int
    L.fsk_b200_tx_engine_new.argtypes = [C.POINTER(TxConfig), C.POINTER(TxSignal), C.c_int]
    L.fsk_b200_tx_engine_new.restype = C.c_void_p
    L.fsk_b200_tx_engine_destroy.argtypes = [C.c_void_p]
    L.fsk_b200_tx_engine_destroy.restype = None
    L.fsk_b200_tx_max_samples.argtypes = [C.c_void_p, C.c_uint32, C.c_uint]
    L.fsk_b200_tx_max_samples.restype = C.c_uint64
    L.fsk_b200_tx_text_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_uint,
                                         C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.fsk_b200_tx_text_batch.restype = C.c_int
    L.fsk_b200_sin_table.argtypes = [C.POINTER(C.c_float), C.c_uint, C.c_float]
    L.fsk_b200_sin_table.restype = None
    L.fsk_b200_version.restype = C.c_char_p
    L.fsk_b200_launch_count.restype = C.c_ulonglong
    L.fsk_b200_last_error.restype = C.c_char_p
    _lib = L
    return L


def version():
    return lib().fsk_b200_version().decode()


def launch_count():
    return int(lib().fsk_b200_launch_count())


def _err(what, rc=None):
    msg = lib().fsk_b200_last_error().decode(errors="replace")
    raise RuntimeError("%s failed%s: %s" % (what, "" if rc is None else " (%d)" % rc, msg))


def rx_config_for_mode(baudmode, sample_rate=48000, **overrides):
    """fsk_b200_rx_config_for_mode: the reference's baudmode presets
    (src/minimodem.c:819-965).  overrides: f_mark, f_space, band_width, n_data_bits,
    nstartbits, nstopbits, inverted, invert_start_stop, msb_first, sync_byte,
    confidence_threshold, confidence_search_limit."""
    ov = RxConfig()
    ov.nstartbits = -1
    ov.nstopbits = -1.0
    for k, v in overrides.items():
        if k == "sync_byte":
            ov.do_rx_sync = 1
            ov.sync_byte = v
        else:
            setattr(ov, k, v)
    out = RxConfig()
    if lib().fsk_b200_rx_config_for_mode(str(baudmode).encode(), float(sample_rate), C.byref(ov),
                                         C.byref(out)) != 0:
        _err("fsk_b200_rx_config_for_mode")
    return out


def rx_params(cfg):
    p = RxParams()
    if lib().fsk_b200_rx_params_derive(C.byref(cfg), C.byref(p)) != 0:
        _err("fsk_b200_rx_params_derive")
    return p


def max_frames(params, nsamples):
    return int(lib().fsk_b200_max_frames(C.byref(params), int(nsamples)))


def frame_databits(params, rec):
    f = Frame(int(rec["bits_lo"]), int(rec["bits_hi"]), float(rec["confidence"]),
              float(rec["amplitude"]), int(rec["frame_start"]))
    return int(lib().fsk_b200_frame_databits(C.byref(params), C.byref(f)))


def sin_table(table_len=4096, amplitude=1.0):
    """The float sine table of the reference tone generator
    (src/simple-tone-generator.c:53-54: mag * sinf((float)M_PI*2*i/len))."""
    out = np.zeros(table_len, np.float32)
    lib().fsk_b200_sin_table(out.ctypes.data_as(C.POINTER(C.c_float)), table_len, amplitude)
    return out


def _torch():
    import torch
    return torch


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream_handle(stream=None):
    torch = _torch()
    s = stream if stream is not None else torch.cuda.current_stream()
    return C.c_void_p(s.cuda_stream)


class FskPlan:
    """Drop-in mirror of the reference's fsk_plan API (src/fsk.h:49-78)."""

    def __init__(self, sample_rate, f_mark, f_space, filter_bw):
        self._p = lib().fsk_plan_new(sample_rate, f_mark, f_space, filter_bw)
        if not self._p:
            raise ValueError("fsk_plan_new() failed")      # NULL + errno, src/fsk.c:58-64

    def __getattr__(self, name):
        if name in ("fftsize", "nbands", "band_width", "b_mark", "b_space", "sample_rate",
                    "f_mark", "f_space"):
            return getattr(self._p.contents, name)
        raise AttributeError(name)

    def find_frame(self, samples, frame_nsamples, try_first_sample, try_max_nsamples,
                   try_step_nsamples, try_confidence_search_limit, expect_bits_string):
        samples = np.ascontiguousarray(samples, np.float32)
        bits, ampl, start = C.c_ulonglong(0), C.c_float(0), C.c_uint(0)
        if isinstance(expect_bits_string, str):
            expect_bits_string = expect_bits_string.encode()
        c = lib().fsk_find_frame(self._p, samples.ctypes.data_as(C.POINTER(C.c_float)), frame_nsamples,
                                 try_first_sample, try_max_nsamples, try_step_nsamples,
                                 try_confidence_search_limit, expect_bits_string,
                                 C.byref(bits), C.byref(ampl), C.byref(start))
        return np.float32(c), bits.value, np.float32(ampl.value), start.value

    def detect_carrier(self, samples, min_mag_threshold):
        samples = np.ascontiguousarray(samples, np.float32)
        return lib().fsk_detect_carrier(self._p, samples.ctypes.data_as(C.POINTER(C.c_float)),
                                        samples.size, min_mag_threshold)

    def set_tones_by_bandshift(self, b_mark, b_shift):
        lib().fsk_set_tones_by_bandshift(self._p, b_mark, b_shift)

    def destroy(self):
        if self._p:
            lib().fsk_plan_destroy(self._p)
            self._p = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


class RxEngine:
    """Batched engine over device-resident streams (Part 2 of include/fsk_b200.h)."""

    def __init__(self, params):
        self.params = params
        self._e = lib().fsk_b200_engine_new(C.byref(params))
        if not self._e:
            _err("fsk_b200_engine_new")

    @classmethod
    def for_mode(cls, baudmode, sample_rate=48000, **overrides):
        return cls(rx_params(rx_config_for_mode(baudmode, sample_rate, **overrides)))

    def tune(self, lanes_per_stream=0, warps_per_block=0, ring_floats=0):
        rc = lib().fsk_b200_engine_tune(self._e, lanes_per_stream, warps_per_block, ring_floats)
        if rc:
            _err("fsk_b200_engine_tune", rc)

    def last_kernel(self):
        """Which rx kernel the latest rx_batch launched (diagnostics)."""
        return lib().fsk_b200_engine_last_kernel(self._e).decode()

    def max_frames(self, nsamples):
        return max_frames(self.params, nsamples)

    def find_frame_batch(self, samples, nvalid, try_first, try_max, try_step, limit,
                         offset=None, expect_sel=None, frames=None, stream=None, bit_mags=False):
        """samples: [nstreams, stride] float32 CUDA tensor; the rest: per-stream CUDA tensors
        (uint32 as int32 storage, float32 limit, uint8 expect_sel).  Returns frames as a
        [nstreams, 5] int32 CUDA tensor (view with frames_to_numpy); with bit_mags=True also a
        [nstreams, n_bits, 2] float32 tensor of the winning candidate's per-bit (signal, noise)
        magnitudes (fsk_b200_find_frame_batch_bits)."""
        torch = _torch()
        assert samples.is_cuda and samples.dtype == torch.float32 and samples.is_contiguous()
        nstreams, stride = samples.shape
        if frames is None:
            frames = torch.empty((nstreams, 5), dtype=torch.int32, device=samples.device)
        if bit_mags:
            mags = torch.zeros((nstreams, self.params.expect_n_bits, 2), dtype=torch.float32, device=samples.device)
            rc = lib().fsk_b200_find_frame_batch_bits(self._e, _ptr(samples), nstreams, stride, _ptr(offset),
                                                      _ptr(nvalid), _ptr(try_first), _ptr(try_max), _ptr(try_step),
                                                      _ptr(limit), _ptr(expect_sel), _ptr(frames), _ptr(mags),
                                                      _stream_handle(stream))
            if rc:
                _err("fsk_b200_find_frame_batch_bits", rc)
            return frames, mags
        rc = lib().fsk_b200_find_frame_batch(self._e, _ptr(samples), nstreams, stride, _ptr(offset),
                                             _ptr(nvalid), _ptr(try_first), _ptr(try_max), _ptr(try_step),
                                             _ptr(limit), _ptr(expect_sel), _ptr(frames),
                                             _stream_handle(stream))
        if rc:
            _err("fsk_b200_find_frame_batch", rc)
        return frames

    def rx_batch(self, samples, nsamples=None, max_frames=None, frames=None, states=None,
                 nsamples_each=None, stream=None):
        """The rx loop over every row of `samples` ([nstreams, stride] float32 CUDA tensor).
        Returns (frames [nstreams, max_frames, 5] int32, states [nstreams, STATE_WORDS] int32)."""
        torch = _torch()
        assert samples.is_cuda and samples.dtype in (torch.float32, torch.int16) and samples.is_contiguous()
        nstreams, stride = samples.shape
        n_all = int(nsamples if nsamples is not None else stride)
        if max_frames is None:
            max_frames = self.max_frames(n_all)
        if frames is None:
            frames = torch.empty((nstreams, max_frames, 5), dtype=torch.int32, device=samples.device)
        if states is None:
            states = torch.zeros((nstreams, STATE_WORDS), dtype=torch.int32, device=samples.device)
        # int16 rows: fsk_b200_rx_batch_s16 (the PCM samples are widened inside the kernel's ring fill)
        fn = lib().fsk_b200_rx_batch if samples.dtype == torch.float32 else lib().fsk_b200_rx_batch_s16
        rc = fn(self._e, _ptr(samples), nstreams, stride, _ptr(nsamples_each), n_all,
                _ptr(frames), max_frames, _ptr(states), _stream_handle(stream))
        if rc:
            _err("fsk_b200_rx_batch", rc)
        return frames, states

    def rx_batch_host(self, samples, nsamples=None, max_frames=None, frames_out=None, states_out=None):
        """Host arrays in, host records out (copies overlap demodulation inside the library).
        samples: [nstreams, stride] float32 numpy array or (pinned) CPU torch tensor;
        frames_out / states_out: optional preallocated host buffers ([n, max_frames, 5] and
        [n, STATE_WORDS] int32 torch tensors, or numpy arrays of FRAME_DTYPE / STATE_DTYPE); states_out
        carries the per-stream state in and out (zero it for fresh streams)."""
        def hptr(t):
            return C.c_void_p(t.data_ptr()) if hasattr(t, "data_ptr") else t.ctypes.data_as(C.c_void_p)
        nstreams, stride = samples.shape
        n_all = int(nsamples if nsamples is not None else stride)
        if max_frames is None:
            max_frames = self.max_frames(n_all)
        if frames_out is None:
            frames_out = np.zeros((nstreams, max_frames), FRAME_DTYPE)
        if states_out is None:
            states_out = np.zeros(nstreams, STATE_DTYPE)
        rc = lib().fsk_b200_rx_batch_host(self._e, hptr(samples), nstreams, stride, n_all,
                                          hptr(frames_out), max_frames, hptr(states_out))
        if rc:
            _err("fsk_b200_rx_batch_host", rc)
        return frames_out, states_out

    def rx_batch_host_s16(self, samples, nsamples=None, max_frames=None, frames_out=None, states_out=None):
        """rx_batch_host for int16 PCM host streams ([nstreams, stride] int16 numpy array or pinned
        CPU torch tensor): half the PCIe bytes, widened to float (x/32768) on the device."""
        def hptr(t):
            return C.c_void_p(t.data_ptr()) if hasattr(t, "data_ptr") else t.ctypes.data_as(C.c_void_p)
        nstreams, stride = samples.shape
        n_all = int(nsamples if nsamples is not None else stride)
        if max_frames is None:
            max_frames = self.max_frames(n_all)
        if frames_out is None:
            frames_out = np.zeros((nstreams, max_frames), FRAME_DTYPE)
        if states_out is None:
            states_out = np.zeros(nstreams, STATE_DTYPE)
        rc = lib().fsk_b200_rx_batch_host_s16(self._e, hptr(samples), nstreams, stride, n_all,
                                              hptr(frames_out), max_frames, hptr(states_out))
        if rc:
            _err("fsk_b200_rx_batch_host_s16", rc)
        return frames_out, states_out

    def decode_ascii_batch(self, frames, states, out_stride=None, stream=None):
        """Device-side databits_decode_ascii8 over the records of rx_batch (CUDA tensors in,
        (bytes [nstreams, out_stride] uint8, counts [nstreams] int32) CUDA tensors out)."""
        torch = _torch()
        nstreams, max_frames = frames.shape[0], frames.shape[1]
        out_stride = int(out_stride or max_frames)
        out = torch.zeros((nstreams, out_stride), dtype=torch.uint8, device=frames.device)
        cnt = torch.zeros((nstreams,), dtype=torch.int32, device=frames.device)
        rc = lib().fsk_b200_decode_ascii_batch(C.byref(self.params), _ptr(frames), _ptr(states), nstreams,
                                               max_frames, _ptr(out), out_stride, _ptr(cnt),
                                               _stream_handle(stream))
        if rc:
            _err("fsk_b200_decode_ascii_batch", rc)
        return out, cnt

    def stream_window(self):
        """fsk_b200_stream_window: the farthest sample a search can touch from its start."""
        return int(lib().fsk_b200_stream_window(C.byref(self.params)))

    def set_holdback(self, nsamples):
        """fsk_b200_engine_set_holdback: searches start only with this many samples left (0 = the
        reference's end-of-input rule)."""
        rc = lib().fsk_b200_engine_set_holdback(self._e, int(nsamples))
        if rc:
            _err("fsk_b200_engine_set_holdback", rc)

    def decode_batch(self, kind, frames, states, dstates=None, out_stride=None, stream=None):
        """Device-side databits decode (N1) of the records of rx_batch with decoder `kind`
        (DECODE_*): CUDA tensors in, (bytes [nstreams, out_stride] uint8, counts [nstreams] int32)
        out.  dstates: uint8 CUDA tensor [nstreams, DECODER_STATE_BYTES] carrying each stream's
        decoder state from batch to batch (updated in place), or None to start from zeros."""
        torch = _torch()
        nstreams, max_frames = frames.shape[0], frames.shape[1]
        if out_stride is None:
            out_stride = decode_max_bytes(kind, self.params.n_data_bits, max_frames)
        out_stride = int(out_stride)
        out = torch.zeros((nstreams, out_stride), dtype=torch.uint8, device=frames.device)
        cnt = torch.zeros((nstreams,), dtype=torch.int32, device=frames.device)
        if dstates is not None:
            assert dstates.dtype == torch.uint8 and tuple(dstates.shape) == (nstreams, DECODER_STATE_BYTES)
        rc = lib().fsk_b200_decode_batch(C.byref(self.params), int(kind), _ptr(frames), _ptr(states), nstreams,
                                         max_frames, _ptr(dstates) if dstates is not None else None,
                                         _ptr(out), out_stride, _ptr(cnt), _stream_handle(stream))
        if rc:
            _err("fsk_b200_decode_batch", rc)
        return out, cnt

    def destroy(self):
        if self._e:
            lib().fsk_b200_engine_destroy(self._e)
            self._e = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


# N1 decoders (include/fsk_b200.h FSK_B200_DECODE_*)
DECODE_ASCII, DECODE_BINARY, DECODE_BAUDOT, DECODE_CALLERID, DECODE_UIC_GROUND, DECODE_UIC_TRAIN = range(6)
DECODER_STATE_BYTES = 272


class DecoderState(C.Structure):
    """fsk_b200_decoder_state"""
    _fields_ = [("baudot_charset", C.c_uint32), ("cid_msgtype", C.c_uint32), ("cid_ndata", C.c_uint32),
                ("reserved", C.c_uint32), ("cid_buf", C.c_uint8 * 256)]


def decoder_for_mode(baudmode, n_data_bits=8, binary_output=False):
    """Which decoder the reference's main() would use (src/minimodem.c:552-892)."""
    k = lib().fsk_b200_decoder_for_mode(str(baudmode).encode(), int(n_data_bits), int(bool(binary_output)))
    if k < 0:
        _err("fsk_b200_decoder_for_mode", k)
    return k


def decode_max_bytes_per_frame(kind, n_data_bits):
    return int(lib().fsk_b200_decode_max_bytes_per_frame(int(kind), int(n_data_bits)))


def detect_carrier_batch(fftsize, samples, nsamples, min_mag_threshold, offset=None, stream=None):
    """fsk_b200_detect_carrier_batch: samples [nstreams, stride] float32 CUDA tensor (optional
    per-stream uint32/int32 `offset` tensor) -> int32 CUDA tensor [nstreams] of band indices (-1 = none)."""
    torch = _torch()
    assert samples.is_cuda and samples.dtype == torch.float32 and samples.is_contiguous()
    nstreams, stride = samples.shape
    out = torch.empty((nstreams,), dtype=torch.int32, device=samples.device)
    rc = lib().fsk_b200_detect_carrier_batch(int(fftsize), _ptr(samples), nstreams, stride, _ptr(offset),
                                             int(nsamples), float(min_mag_threshold), _ptr(out),
                                             _stream_handle(stream))
    if rc:
        _err("fsk_b200_detect_carrier_batch", rc)
    return out


def stream_push(rows, fill, states, chunk, chunk_len=None, dropped=None, stream=None):
    """fsk_b200_stream_push on CUDA tensors: rows [n, stride] float32, fill [n] int32 (in/out), states
    [n, STATE_WORDS] int32 (in/out), chunk [n, chunk_stride] float32, chunk_len [n] int32 or an int."""
    torch = _torch()
    # the C call takes raw pointers and row strides: the tensors must be what it assumes
    assert rows.is_contiguous() and rows.dtype == torch.float32 and chunk.is_contiguous() and chunk.dtype == torch.float32
    assert fill.is_contiguous() and fill.dtype == torch.int32 and states.is_contiguous() and states.dtype == torch.int32
    assert chunk.shape[0] == rows.shape[0] and states.shape == (rows.shape[0], STATE_WORDS)
    n, stride = rows.shape
    per = chunk_len if hasattr(chunk_len, "data_ptr") else None
    assert per is None or (per.dtype == torch.int32 and per.is_contiguous())
    common = 0 if per is not None else int(chunk.shape[1] if chunk_len is None else chunk_len)
    rc = lib().fsk_b200_stream_push(_ptr(rows), n, stride, _ptr(fill), _ptr(states), _ptr(chunk),
                                    chunk.shape[1], _ptr(per), common, _ptr(dropped), _stream_handle(stream))
    if rc:
        _err("fsk_b200_stream_push", rc)


def wav_locate(image):
    """fsk_b200_wav_locate on a bytes object: (data_offset, nsamples, sample_rate, is_float)."""
    off, n, rate, isf = C.c_size_t(0), C.c_size_t(0), C.c_uint32(0), C.c_int(0)
    rc = lib().fsk_b200_wav_locate(image, len(image), C.byref(off), C.byref(n), C.byref(rate), C.byref(isf))
    if rc:
        _err("fsk_b200_wav_locate", rc)
    return off.value, n.value, rate.value, bool(isf.value)


def decode_max_bytes(kind, n_data_bits, nframes):
    """out_stride that never truncates `nframes` records of one stream."""
    return int(lib().fsk_b200_decode_max_bytes(int(kind), int(n_data_bits), int(nframes)))


def frames_to_numpy(frames):
    """int32 CUDA/CPU tensor [..., 5] -> structured numpy records."""
    a = frames.detach().cpu().numpy()
    return np.ascontiguousarray(a).view(FRAME_DTYPE).reshape(a.shape[:-1])


def check_not_truncated(states, max_frames):
    """Raises if a stream stopped because its record buffer was full (done == 0 and nframes == max_frames,
    include/fsk_b200.h): its decode is incomplete until the caller consumes the records, resets nframes and
    calls rx_batch again.  Synchronises (reads the states back)."""
    st = states_to_numpy(states)
    bad = np.nonzero((st["done"] == 0) & (st["nframes"] >= int(max_frames)))[0]
    if bad.size:
        raise RuntimeError("rx_batch: %d stream(s) filled their %d-record buffer before the end of their samples "
                           "(first: stream %d); use RxEngine.max_frames(nsamples) or resume them" % (
                               bad.size, int(max_frames), int(bad[0])))


def states_to_numpy(states):
    a = states.detach().cpu().numpy()
    return np.ascontiguousarray(a).view(STATE_DTYPE).reshape(a.shape[:-1])


def tx_batch(cfg, words, nsamples_out, lead_in=None, table=None, out=None, stride=None, stream=None):
    """Device-side synthesis of test streams (fsk_b200_tx_batch).  words: [nstreams, nwords]
    int32 CUDA tensor; table: float32 CUDA tensor (default: the reference's 4096-entry
    float sine table).  Returns [nstreams, stride] float32 CUDA tensor."""
    torch = _torch()
    nstreams, nwords = words.shape
    if table is None:
        table = torch.from_numpy(sin_table()).to(words.device)
    if stride is None:
        stride = (int(nsamples_out) + 3) & ~3
    if out is None:
        out = torch.empty((nstreams, stride), dtype=torch.float32, device=words.device)
    rc = lib().fsk_b200_tx_batch(C.byref(cfg), _ptr(table), table.numel(), _ptr(words), nwords,
                                 _ptr(lead_in), _ptr(out), nstreams, stride, int(nsamples_out),
                                 _stream_handle(stream))
    if rc:
        _err("fsk_b200_tx_batch", rc)
    return out


def s16_to_f32(src, out=None, stream=None):
    """[nstreams, stride] int16 CUDA tensor -> float32 (x/32768) on the device."""
    torch = _torch()
    nstreams, stride = src.shape
    if out is None:
        out = torch.empty((nstreams, stride), dtype=torch.float32, device=src.device)
    rc = lib().fsk_b200_s16_to_f32(_ptr(src), _ptr(out), nstreams, stride, _stream_handle(stream))
    if rc:
        _err("fsk_b200_s16_to_f32", rc)
    return out


def tx_config_from(cfg, leader_bits=None, trailer_bits=2, do_tx_sync_bytes=None):
    """TxConfig matching an RxConfig (fsk_b200_tx_config_from_rx: what src/minimodem.c:716-720, :844-845,
    :949-951 derive); the keywords override its fields."""
    t = TxConfig()
    if lib().fsk_b200_tx_config_from_rx(C.byref(cfg), C.byref(t)) != 0:
        _err("fsk_b200_tx_config_from_rx")
    if do_tx_sync_bytes is not None:
        t.do_tx_sync_bytes = do_tx_sync_bytes
    if leader_bits is not None:
        t.leader_bits = leader_bits
    t.trailer_bits = trailer_bits
    return t


def encoder_for_mode(baudmode, n_data_bits=8):
    """Which databits encoder the reference's main() would use (ENCODE_ASCII8 / ENCODE_BAUDOT)."""
    k = lib().fsk_b200_encoder_for_mode(str(baudmode).encode(), int(n_data_bits))
    if k < 0:
        _err("fsk_b200_encoder_for_mode", k)
    return k


class TxEngine:
    """The batched transmitter (fsk_b200_tx_engine): text rows in, the reference's `--tx` samples out,
    all on the device.  cfg: TxConfig; the signal options are --volume, --lut and --float-samples."""

    def __init__(self, cfg, encoder=ENCODE_ASCII8, amplitude=1.0, lut=4096, float_samples=False):
        self.cfg = cfg
        self.encoder = int(encoder)
        self.float_samples = bool(float_samples)
        sig = TxSignal(float(amplitude), int(lut), int(self.float_samples))
        self._te = lib().fsk_b200_tx_engine_new(C.byref(cfg), C.byref(sig), self.encoder)
        if not self._te:
            _err("fsk_b200_tx_engine_new")

    @classmethod
    def for_mode(cls, baudmode, sample_rate=48000, amplitude=1.0, lut=4096, float_samples=False, **overrides):
        rx = rx_config_for_mode(baudmode, sample_rate, **overrides)
        return cls(tx_config_from(rx), encoder_for_mode(baudmode, rx.n_data_bits), amplitude, lut, float_samples)

    def max_samples(self, nbytes, flags=0):
        """fsk_b200_tx_max_samples: the out_stride a row of nbytes text bytes never exceeds."""
        return int(lib().fsk_b200_tx_max_samples(self._te, int(nbytes), int(flags)))

    def new_states(self, nstreams, device=None):
        """Fresh per-stream states: uint8 CUDA tensor [nstreams, TX_STATE_BYTES] of zeros."""
        torch = _torch()
        return torch.zeros((int(nstreams), TX_STATE_BYTES), dtype=torch.uint8,
                           device=device if device is not None else torch.device("cuda:0"))

    def text_batch(self, text, lengths, states, flags=0, out=None, out_len=None, stream=None):
        """fsk_b200_tx_text_batch.  text: uint8 CUDA tensor [nstreams, text_stride]; lengths: int32
        [nstreams]; states: uint8 [nstreams, TX_STATE_BYTES] (updated in place).  Returns (samples
        [nstreams, out_stride] int16 or float32, counts [nstreams] int32)."""
        torch = _torch()
        assert text.dtype == torch.uint8 and text.is_contiguous() and text.dim() == 2
        nstreams, text_stride = text.shape
        assert lengths.dtype == torch.int32 and lengths.is_contiguous() and lengths.numel() == nstreams
        assert states.dtype == torch.uint8 and states.is_contiguous() and tuple(states.shape) == (nstreams, TX_STATE_BYTES)
        if out is None:
            stride = (self.max_samples(text_stride, flags) + 7) & ~7
            out = torch.empty((nstreams, stride), dtype=torch.float32 if self.float_samples else torch.int16,
                              device=text.device)
        assert out.is_contiguous() and out.dtype == (torch.float32 if self.float_samples else torch.int16)
        if out_len is None:
            out_len = torch.empty((nstreams,), dtype=torch.int32, device=text.device)
        rc = lib().fsk_b200_tx_text_batch(self._te, _ptr(text), nstreams, text_stride, _ptr(lengths), int(flags),
                                          _ptr(states), _ptr(out), out.shape[1], _ptr(out_len),
                                          _stream_handle(stream))
        if rc:
            _err("fsk_b200_tx_text_batch", rc)
        return out, out_len

    def destroy(self):
        if self._te:
            lib().fsk_b200_tx_engine_destroy(self._te)
            self._te = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


def tx_max_samples(engine, nbytes, flags=0):
    """fsk_b200_tx_max_samples of a TxEngine."""
    return engine.max_samples(nbytes, flags)
