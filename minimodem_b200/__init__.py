"""minimodem_b200 -- H100-native (sm_90a) batched FSK demodulation engine.

The product is the C-ABI shared library ``libfsk_b200.so`` (include/fsk_b200.h):
C host code + hand-written CUDA kernels for sm_90a.  This package is the thin
Python binding over that ABI (ctypes; torch only provides device memory,
streams and torch.distributed).  There is no CPU or PyTorch fallback: importing
works anywhere, but every analysis call needs the library and a CUDA device and
raises otherwise.
"""
from .api import (  # noqa: F401
    LIB_PATH, Frame, RxConfig, RxParams, RxEngine, FskPlan, StreamState, TxConfig,
    build, lib, rx_config_for_mode, rx_params, frame_databits, max_frames, tx_batch,
    version, launch_count, sin_table, frames_to_numpy, states_to_numpy, check_not_truncated, tx_config_from, s16_to_f32,
    FRAME_DTYPE, STATE_DTYPE, STATE_WORDS, FRAME_ACQUIRED, FRAME_REPORT, EXPORTS,
    DECODE_ASCII, DECODE_BINARY, DECODE_BAUDOT, DECODE_CALLERID, DECODE_UIC_GROUND, DECODE_UIC_TRAIN,
    DECODER_STATE_BYTES, DecoderState, decoder_for_mode, decode_max_bytes_per_frame, decode_max_bytes, detect_carrier_batch, stream_push, wav_locate,
    TxEngine, TxSignal, TxState, TX_STATE_BYTES, TX_IDLE_IF_EMPTY, TX_FINAL, ENCODE_ASCII8, ENCODE_BAUDOT,
    encoder_for_mode, tx_max_samples,
)
from .serving import LiveReceiver, LiveTransmitter  # noqa: F401,E402
