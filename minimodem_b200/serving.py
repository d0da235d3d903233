"""A receiver and a transmitter for live streams, composed from the C ABI's batched calls
(include/fsk_b200.h):

    rx = LiveReceiver("rtty", sample_rate=8000, nstreams=4096, max_chunk=2000)
    for chunk, lengths in source:                 # float32 CUDA tensor [nstreams, <= max_chunk]
        text, counts = rx.feed(chunk, lengths)    # uint8 CUDA tensor [nstreams, row], int32 [nstreams]
    text, counts = rx.finish()

Per call: fsk_b200_stream_push (carry the unconsumed tail, append the chunk) -> fsk_b200_rx_batch
(the whole rx loop, src/minimodem.c:1137-1463) -> fsk_b200_decode_batch (the reference's databits
decoder for the mode, with its per-stream state carried along).  The holdback is set so that a
search only starts when every sample it can touch has arrived: the text does not depend on how
the stream was cut into chunks (tests/test_gpu_parity.py::test_live_receiver_*).  Everything
stays on the device; there is no per-stream work on the host.

    tx = LiveTransmitter("rtty", sample_rate=8000, nstreams=4096, max_text=64)
    for text, lengths in source:                  # uint8 CUDA tensor [nstreams, <= max_text], int32 [nstreams]
        audio, counts = tx.feed(text, lengths)    # int16 (or float32) CUDA tensor [nstreams, row], int32 [nstreams]
    audio, counts = tx.finish()                   # the trailers

Per call one fsk_b200_tx_text_batch: the reference transmitter (src/minimodem.c:114-250) for each
stream's bytes, its tone phase, Baudot charset and carrier state carried on the device, so the
audio does not depend on how the text was cut into feeds.  With idle=True a stream that has no
bytes in a feed sends the reference's idle tone, as the reference does when its input pipe pauses."""
import ctypes as C

from . import api


class LiveReceiver:
    def __init__(self, baudmode, sample_rate=48000, nstreams=1, max_chunk=4800, device=None,
                 binary_output=False, **overrides):
        torch = api._torch()
        cfg = api.rx_config_for_mode(baudmode, sample_rate, **overrides)
        self.engine = api.RxEngine(api.rx_params(cfg))
        self.kind = api.decoder_for_mode(baudmode, self.engine.params.n_data_bits, binary_output)
        self.window = self.engine.stream_window()
        self.engine.set_holdback(self.window)
        self.nstreams, self.max_chunk = int(nstreams), int(max_chunk)
        # a row holds the longest tail the loop can leave behind plus one chunk
        tail_max = self.window + self.engine.params.frame_nsamples
        self.stride = (tail_max + self.max_chunk + 3) & ~3
        self.max_frames = self.engine.max_frames(self.stride)
        self.row_bytes = api.decode_max_bytes(self.kind, self.engine.params.n_data_bits, self.max_frames)
        dev = device if device is not None else torch.device("cuda:0")
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
        self.rows = z((self.nstreams, self.stride), torch.float32)
        self.fill = z((self.nstreams,), torch.int32)
        self.states = z((self.nstreams, api.STATE_WORDS), torch.int32)
        self.dstates = z((self.nstreams, api.DECODER_STATE_BYTES), torch.uint8)
        self.dropped = z((self.nstreams,), torch.int32)
        self._empty = z((self.nstreams, 4), torch.float32)

    def _step(self, chunk, lengths):
        api.stream_push(self.rows, self.fill, self.states, chunk, lengths, dropped=self.dropped)
        frames, self.states = self.engine.rx_batch(self.rows, nsamples=self.stride, nsamples_each=self.fill,
                                                   max_frames=self.max_frames, states=self.states)
        return self.engine.decode_batch(self.kind, frames, self.states, dstates=self.dstates,
                                        out_stride=self.row_bytes)

    def feed(self, chunk, lengths=None):
        """chunk: float32 CUDA tensor [nstreams, width <= max_chunk]; lengths: int32 CUDA tensor [nstreams]
        (samples valid in each row of the chunk) or None = the whole width.  Returns (text, counts)."""
        assert chunk.shape[0] == self.nstreams and chunk.shape[1] <= self.max_chunk
        return self._step(chunk, lengths)

    def finish(self):
        """End of input: the reference's rule (it analyses what is left while expect_nsamples remain,
        src/minimodem.c:1229) replaces the holdback for one last pass."""
        self.engine.set_holdback(0)
        out = self._step(self._empty, 0)
        self.engine.set_holdback(self.window)
        return out


class LiveTransmitter:
    def __init__(self, baudmode, sample_rate=48000, nstreams=1, max_text=256, float_samples=False, amplitude=1.0,
                 lut=4096, idle=True, device=None, **overrides):
        torch = api._torch()
        self.engine = api.TxEngine.for_mode(baudmode, sample_rate, amplitude, lut, float_samples, **overrides)
        self.nstreams, self.max_text = int(nstreams), int(max_text)
        self.flags = api.TX_IDLE_IF_EMPTY if idle else 0
        dev = device if device is not None else torch.device("cuda:0")
        self.states = self.engine.new_states(self.nstreams, dev)
        self._empty = torch.zeros((self.nstreams, 1), dtype=torch.uint8, device=dev)
        self._zero = torch.zeros((self.nstreams,), dtype=torch.int32, device=dev)

    def feed(self, text, lengths=None):
        """text: uint8 CUDA tensor [nstreams, width <= max_text]; lengths: int32 CUDA tensor [nstreams]
        (bytes valid in each row) or None = the whole width.  Returns (audio, counts): audio row s holds
        counts[s] samples."""
        torch = api._torch()
        assert text.shape[0] == self.nstreams and text.shape[1] <= self.max_text
        if lengths is None:
            lengths = torch.full((self.nstreams,), text.shape[1], dtype=torch.int32, device=text.device)
        return self.engine.text_batch(text.contiguous(), lengths, self.states, self.flags)

    def finish(self):
        """End of input: every stream that is transmitting sends the trailer (src/minimodem.c:246-249)."""
        return self.engine.text_batch(self._empty, self._zero, self.states, api.TX_FINAL)
