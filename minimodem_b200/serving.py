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
stays on the device; there is no per-stream work on the host.  With auto_carrier=threshold (0.001 is
the CLI's -a) every stream finds its own tone pair: fsk_b200_rx_batch_auto with the per-stream
auto states and the auto holdback (fsk_b200_auto_stream_window) in place of fsk_b200_rx_batch.
With tones=bands (an int32 tensor [nstreams, 2] from RxEngine.tone_bands on an engine of the same mode,
or rx.engine.tone_bands) every stream keeps its own -M / -S pair: fsk_b200_rx_batch_tones with the
ordinary holdback; tones and auto_carrier exclude each other.  With channels_per_row=k and tones [nstreams*k, 2]
each fed row carries k channels (both directions of a duplex line, k signals of a passband): one push per row
(fsk_b200_stream_push_channels, where a disabled channel does not hold the row back), one
fsk_b200_rx_batch_channels, and text and decoder state per channel, [nstreams*k, ...].

With pcm16=True the receiver takes int16 CUDA chunks (16-bit PCM, LiveTransmitter's default output) in every form above:
the rows stay int16 (stride a multiple of 8), the push is fsk_b200_stream_push_s16 and the rx call its _s16 form, widened
(x / 32768, exact) inside the kernel's ring fill; the text is the float receiver's on the widened chunks.  Where
fsk_b200_rx_batch_s16_runs says the plain int16 call has no build for the mode, the rows are float32 and every chunk is
widened into a preallocated buffer before the float push; rx.rows.dtype shows which.

Streams with lifetimes of their own (calls on a modem bank, a Caller-ID front end):

    text, counts = rx.feed(chunk, lengths, opened=opened, ended=ended)   # bool CUDA tensors [nstreams]

In one feed the opened rows start a new stream (their decoder and auto states zeroed on the device), every
row's chunk is pushed with the row events of fsk_b200_stream_push_events, and an ended row (this chunk is its
last) comes back decoded to its end by the reference's end-of-input rule while the other rows stay held back.
A row that ended in an earlier feed and is not reopened returns count 0; its chunk is counted in rx.dropped,
and its final state (with the carrier session still open at its end) stays in rx.states until it is reopened.

    tx = LiveTransmitter("rtty", sample_rate=8000, nstreams=4096, max_text=64)
    for text, lengths in source:                  # uint8 CUDA tensor [nstreams, <= max_text], int32 [nstreams]
        audio, counts = tx.feed(text, lengths)    # int16 (or float32) CUDA tensor [nstreams, row], int32 [nstreams]
    audio, counts = tx.finish()                   # the trailers

Per call one fsk_b200_tx_text_batch: the reference transmitter (src/minimodem.c:114-250) for each
stream's bytes, its tone phase, Baudot charset and carrier state carried on the device, so the
audio does not depend on how the text was cut into feeds.  With idle=True a stream that has no
bytes in a feed sends the reference's idle tone, as the reference does when its input pipe pauses.
With tones=pairs (a float32 tensor [nstreams, 2] from TxEngine.tone_pairs) every stream sends on its own
-M / -S pair: fsk_b200_tx_text_batch_tones, the tensor read at every feed and at finish."""
import ctypes as C

from . import api


class LiveReceiver:
    def __init__(self, baudmode, sample_rate=48000, nstreams=1, max_chunk=4800, device=None,
                 binary_output=False, auto_carrier=None, tones=None, channels_per_row=1, pcm16=False, **overrides):
        torch = api._torch()
        if auto_carrier is not None and tones is not None:
            raise ValueError("LiveReceiver: auto_carrier and tones exclude each other")
        self.k = int(channels_per_row)
        if self.k != 1 and tones is None:
            raise ValueError("LiveReceiver: channels_per_row needs tones, a pair per channel")
        self.engine = api.RxEngine.for_mode(baudmode, sample_rate, **overrides)
        self.kind = api.decoder_for_mode(baudmode, self.engine.params.n_data_bits, binary_output)
        self.auto = auto_carrier is not None
        if self.auto:
            self.engine.set_auto_carrier(auto_carrier, inverted=bool(overrides.get("inverted", False)))
        self.window = self.engine.auto_stream_window() if self.auto else self.engine.stream_window()
        self.engine.set_holdback(self.window)
        self.nstreams, self.max_chunk = int(nstreams), int(max_chunk)
        # a row holds the longest tail the loop can leave behind plus one chunk
        tail_max = self.window + self.engine.params.frame_nsamples
        self.pcm16 = bool(pcm16)
        align = 8 if self.pcm16 else 4         # int16 rows: the row layout of the _s16 calls
        self.stride = (tail_max + self.max_chunk + align - 1) & ~(align - 1)
        self.max_frames = self.engine.max_frames(self.stride)
        self.row_bytes = api.decode_max_bytes(self.kind, self.engine.params.n_data_bits, self.max_frames)
        dev = device if device is not None else torch.device("cuda:0")
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
        nchannels = self.nstreams * self.k
        # pcm16: int16 rows wherever the rx call has an int16 build (the tone and auto-carrier calls always do);
        # elsewhere float32 rows, and every chunk is widened exactly (x / 32768) before the push
        s16_rows = self.pcm16 and (tones is not None or self.auto or self.engine.rx_batch_s16_runs(self.nstreams))
        row_type = torch.int16 if s16_rows else torch.float32
        self.rows = z((self.nstreams, self.stride), row_type)
        self.fill = z((self.nstreams,), torch.int32)
        self.states = z((nchannels, api.STATE_WORDS), torch.int32)
        self.dstates = z((nchannels, api.DECODER_STATE_BYTES), torch.uint8)
        self.dropped = z((self.nstreams,), torch.int32)
        self._empty = z((self.nstreams, align), row_type)
        self._wide = self._stage = None
        if self.pcm16 and not s16_rows:
            # flat buffers, viewed [nstreams, width] per chunk: 16-byte aligned, contiguous at every width
            wide = (self.max_chunk + 3) & ~3
            self._wide = z((self.nstreams * wide,), torch.float32)
            self._stage = z((self.nstreams * wide,), torch.int16)
        self.auto_states = z((self.nstreams, api.AUTO_STATE_BYTES), torch.uint8) if self.auto else None
        self.tones = None
        if tones is not None:
            assert tuple(tones.shape) == (nchannels, 2)
            self.tones = tones.to(device=dev, dtype=torch.int32).contiguous()
        self._ended = None          # bool [nstreams]: rows whose stream has ended, once events are in use

    def _step(self, chunk, lengths, events=None):
        if events is None and self._ended is not None:
            # once rows have ended, every push carries events, so that their flag survives
            events = self._no_events
        if self.k > 1 or events is not None:
            api.stream_push(self.rows, self.fill, self.states, chunk, lengths, dropped=self.dropped,
                            channels_per_row=self.k, tone_bands=self.tones, nbands=self.engine.params.nbands,
                            row_events=events)
        else:
            api.stream_push(self.rows, self.fill, self.states, chunk, lengths, dropped=self.dropped)
        if self.tones is not None:
            frames, self.states = self.engine.rx_batch_tones(
                self.rows, self.tones, nsamples=self.stride, nsamples_each=self.fill, max_frames=self.max_frames,
                states=self.states, channels_per_row=self.k)
        elif self.auto:
            frames, self.states, self.auto_states = self.engine.rx_batch_auto(
                self.rows, nsamples=self.stride, nsamples_each=self.fill, max_frames=self.max_frames,
                states=self.states, auto_states=self.auto_states)
        else:
            frames, self.states = self.engine.rx_batch(self.rows, nsamples=self.stride, nsamples_each=self.fill,
                                                       max_frames=self.max_frames, states=self.states)
        states = self.states
        if self._ended is not None:
            # rows that ended in an earlier feed: the rx call skipped them, and their records were decoded then
            torch = api._torch()
            stale = self._ended.repeat_interleave(self.k)
            states = torch.where(stale[:, None] & self._nframes_word, 0, self.states)
        return self.engine.decode_batch(self.kind, frames, states, dstates=self.dstates,
                                        out_stride=self.row_bytes)

    def _widened(self, chunk):
        """the int16 chunk as float32 (x / 32768, exact) in the preallocated buffer, for float rows"""
        n, w = chunk.shape
        w4 = (w + 3) & ~3
        src = chunk
        if w4 != w or not chunk.is_contiguous() or chunk.data_ptr() % 8:
            src = self._stage[:n * w4].view(n, w4)     # fsk_b200_s16_to_f32 takes strides of 4 samples
            src[:, :w].copy_(chunk)
        out = self._wide[:n * w4].view(n, w4)
        api.s16_to_f32(src, out=out)
        return out

    def feed(self, chunk, lengths=None, opened=None, ended=None):
        """chunk: float32 CUDA tensor [nstreams, width <= max_chunk] (int16 with pcm16=True); lengths: int32 CUDA
        tensor [nstreams] (samples valid in each row of the chunk) or None = the whole width.  opened / ended:
        bool CUDA tensors [nstreams] or None: rows where a new stream starts with this chunk, rows whose stream
        ends with it (both: a whole stream in one chunk).  Returns (text, counts)."""
        assert chunk.shape[0] == self.nstreams and chunk.shape[1] <= self.max_chunk
        torch = api._torch()
        want = torch.int16 if self.pcm16 else torch.float32
        if chunk.dtype != want:
            raise TypeError("LiveReceiver.feed: a %s chunk, this receiver takes %s" % (chunk.dtype, want))
        if lengths is None:
            lengths = chunk.shape[1]
        if self._wide is not None:
            chunk = self._widened(chunk)
        if opened is None and ended is None:
            return self._step(chunk, lengths)
        dev = self.rows.device
        no = torch.zeros((self.nstreams,), dtype=torch.bool, device=dev)
        opened = no if opened is None else opened.to(device=dev, dtype=torch.bool)
        ended = no if ended is None else ended.to(device=dev, dtype=torch.bool)
        assert tuple(opened.shape) == (self.nstreams,) and tuple(ended.shape) == (self.nstreams,)
        if self._ended is None:
            self._ended = no.clone()
            self._nframes_word = torch.zeros((1, api.STATE_WORDS), dtype=torch.bool, device=dev)
            self._nframes_word[0, 2] = True         # StreamState.nframes
            self._no_events = torch.zeros((self.nstreams,), dtype=torch.uint8, device=dev)
        # the push owns the stream states of an opened row; the decoder and auto states are zeroed here
        self.dstates.masked_fill_(opened.repeat_interleave(self.k)[:, None], 0)
        if self.auto:
            self.auto_states.masked_fill_(opened[:, None], 0)
        self._ended &= ~opened
        events = opened.to(torch.uint8) * api.ROW_OPEN + ended.to(torch.uint8) * api.ROW_END
        out = self._step(chunk, lengths, events)
        self._ended |= ended
        return out

    def finish(self):
        """End of input: the reference's rule (it analyses what is left while expect_nsamples remain,
        src/minimodem.c:1229) replaces the holdback for one last pass."""
        self.engine.set_holdback(0)
        out = self._step(self._empty, 0)
        self.engine.set_holdback(self.window)
        return out


class LiveTransmitter:
    def __init__(self, baudmode, sample_rate=48000, nstreams=1, max_text=256, float_samples=False, amplitude=1.0,
                 lut=4096, idle=True, device=None, tones=None, **overrides):
        torch = api._torch()
        self.engine = api.TxEngine.for_mode(baudmode, sample_rate, amplitude, lut, float_samples, **overrides)
        self.nstreams, self.max_text = int(nstreams), int(max_text)
        self.flags = api.TX_IDLE_IF_EMPTY if idle else 0
        dev = device if device is not None else torch.device("cuda:0")
        self.states = self.engine.new_states(self.nstreams, dev)
        self._empty = torch.zeros((self.nstreams, 1), dtype=torch.uint8, device=dev)
        self._zero = torch.zeros((self.nstreams,), dtype=torch.int32, device=dev)
        # float32 [nstreams, 2] (TxEngine.tone_pairs): kept by reference and read at every call, so a caller
        # may move a stream to another pair between feeds by writing into it
        self.tones = None
        if tones is not None:
            assert tuple(tones.shape) == (self.nstreams, 2) and tones.dtype == torch.float32 and tones.is_contiguous()
            self.tones = tones

    def feed(self, text, lengths=None):
        """text: uint8 CUDA tensor [nstreams, width <= max_text]; lengths: int32 CUDA tensor [nstreams]
        (bytes valid in each row) or None = the whole width.  Returns (audio, counts): audio row s holds
        counts[s] samples."""
        torch = api._torch()
        assert text.shape[0] == self.nstreams and text.shape[1] <= self.max_text
        if lengths is None:
            lengths = torch.full((self.nstreams,), text.shape[1], dtype=torch.int32, device=text.device)
        return self.engine.text_batch(text.contiguous(), lengths, self.states, self.flags, tones=self.tones)

    def finish(self):
        """End of input: every stream that is transmitting sends the trailer (src/minimodem.c:246-249)."""
        return self.engine.text_batch(self._empty, self._zero, self.states, api.TX_FINAL, tones=self.tones)
