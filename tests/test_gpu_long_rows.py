"""Rows that end near the 32-bit sample-position limit (FSK_B200_MAX_ROW_SAMPLES = 2^32 - 4).

Positions inside a row are 32-bit, and the kernels add to them: the request limits of the ring fill, the
end of a search window, the tail blocks and the generic kernels' sample indices.  A sum that wraps near
2^32 reads the row's start, or takes the zeros past the row's end for samples, and the kernel still
writes a plausible record.  So every rx kernel family here decodes a stream placed at the END of a long
row and the same samples at the start of a small row, and the two must agree: records byte for byte,
every byte of the state except `pos`, which differs by exactly the distance between the two placements.

A long row costs megabytes, not 16 GB: the fixture reserves the whole range of two rows of 2^32 samples
and maps ONE physical body chunk at every chunk of it, with separate real chunks where a stream lives and
for a guard past the second row.  On the GPU through the driver's virtual-memory calls (cuMemCreate /
cuMemAddressReserve / cuMemMap), under FSK_B200_EMU=1 with a memfd mapped over a PROT_NONE reservation.
The physical footprint is 17 chunks of 4 MB, 68 MB in all (the module fixture checks it stays under 128 MB).  Every chunk holds loud noise
plus an in-band tone, never zeros: a wrapped index that reads the row's start, or a fill that reads past
the row's end instead of storing zeros, changes a record.  The whole range is mapped, so a wrapped read
gives wrong records and never faults.

Also here: the rx calls refuse nsamples_all above the limit with nothing launched, the live push caps a
row at the limit, and the transmitter's lead-in and length bounds at 2^32 - 1."""
import ctypes as C
import os

import numpy as np
import pytest

import autoorc
import minimodem_b200 as mm
import orc
import rxfam
import tie_screen
from gpudev import dev, emulated, pcm, sync, torch, upload
from rxfam import as_oracle_frames, compare_frames, compare_reports, reports_of

pytestmark = pytest.mark.gpu

TOP = 1 << 32
MAX_ROW = TOP - 4
STRIDE = TOP                    # elements per row of the long layout (a multiple of 8)
CHUNK = 4 << 20                 # bytes per mapped chunk (a multiple of the H100's 2 MB granularity)
GUARD = 2 << 20                 # bytes of real memory past the second row
HOT_BEFORE, HOT_AFTER = 300_000, 60_000     # samples around a row end that get their own chunks

# row lengths: 2^32 - 4 and every n mod 8 below it, the last ring blocks, the sign boundary, a control
TOPS = [4, 5, 6, 7, 8, 11] + [4 + d for d in (16, 64, 128, 256, 1024)]
ROW_LENGTHS = [("top%d" % d, TOP - d) for d in TOPS] + [
    ("sign-1", (1 << 31) - 1), ("sign0", 1 << 31), ("sign+1", (1 << 31) + 1), ("ctrl20", 1 << 20)]
CASES = ("at-start", "earlier", "cut")


# ---------------------------------------------------------------------------------------------------
# the aliased rows
# ---------------------------------------------------------------------------------------------------
def hot_ranges():
    """sample ranges [lo, hi) of row 0 and row 1 that need memory of their own"""
    r = []
    for _, n in ROW_LENGTHS:
        r.append((n - HOT_BEFORE, n + HOT_AFTER))
    r.append((STRIDE + MAX_ROW - HOT_BEFORE, STRIDE + MAX_ROW + HOT_AFTER))
    return r


class _Driver:
    """the CUDA driver's virtual-memory calls through ctypes"""

    def __init__(self):
        self.cu = C.CDLL("libcuda.so.1")
        for name in ("cuMemAddressReserve", "cuMemAddressFree", "cuMemCreate", "cuMemRelease", "cuMemMap",
                     "cuMemUnmap", "cuMemSetAccess", "cuMemGetAllocationGranularity", "cuCtxGetDevice",
                     "cuMemGetInfo_v2", "cuMemGetAddressRange_v2"):
            getattr(self.cu, name).restype = C.c_int

    def ok(self, rc, what):
        assert rc == 0, "%s: CUresult %d" % (what, rc)

    def device(self):
        d = C.c_int()
        self.ok(self.cu.cuCtxGetDevice(C.byref(d)), "cuCtxGetDevice")
        return d.value

    def prop(self, dev):
        # CUmemAllocationProp: type PINNED, no handle type, location (DEVICE, dev), meta, flags
        p = (C.c_ubyte * 32)()
        C.memmove(p, np.array([1, 0, 1, dev], np.int32).tobytes(), 16)
        return p

    def mem_info(self):
        free, total = C.c_size_t(), C.c_size_t()
        self.ok(self.cu.cuMemGetInfo_v2(C.byref(free), C.byref(total)), "cuMemGetInfo")
        return free.value, total.value


class AliasedRows:
    """[rows, STRIDE] samples of `dtype` over one physical body chunk, real chunks over hot_ranges() and a
    guard past the last row; .t is the tensor, .close() undoes every mapping"""

    def __init__(self, dtype, rows=2):
        self.dtype = np.dtype(dtype)
        self.es = self.dtype.itemsize
        self.nbytes = -(-(rows * STRIDE * self.es + GUARD) // CHUNK) * CHUNK
        nchunks = self.nbytes // CHUNK
        hot = set()
        for lo, hi in hot_ranges():
            hot.update(range(max(lo, 0) * self.es // CHUNK, min(hi * self.es // CHUNK, nchunks - 1) + 1))
        hot.update(range((rows * STRIDE * self.es) // CHUNK, nchunks))        # the guard
        self.hot = sorted(hot)
        self.body = next(i for i in range(nchunks) if i not in hot)
        self.physical = (1 + len(self.hot)) * CHUNK
        self.emu = emulated()
        self._map(nchunks)
        t = torch()
        nel = self.nbytes // self.es            # the rows and the guard behind them
        if self.emu:
            arr = np.ctypeslib.as_array(C.cast(self.base, C.POINTER(np.ctypeslib.as_ctypes_type(self.dtype))),
                                        shape=(nel,))
            self.flat = t.from_numpy(arr)
        else:
            class _Cai:
                pass
            o = _Cai()
            o.__cuda_array_interface__ = dict(shape=(nel,), typestr=self.dtype.str, data=(self.base, False),
                                              strides=None, version=2)
            self.flat = t.as_tensor(o, device=dev())
        self.t = self.flat[:rows * STRIDE].view(rows, STRIDE)
        rng = np.random.default_rng(99 + self.es)
        for ci in [self.body] + self.hot:
            e0, ne = ci * CHUNK // self.es, CHUNK // self.es
            self.write(e0, loud(rng, ne, self.dtype))

    def _map(self, nchunks):
        if self.emu:
            libc = C.CDLL(None, use_errno=True)
            libc.mmap.restype = C.c_void_p
            libc.mmap.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_long]
            libc.munmap.argtypes = [C.c_void_p, C.c_size_t]
            self.libc = libc
            base = libc.mmap(None, self.nbytes, 0, 0x02 | 0x20 | 0x4000, -1, 0)   # PROT_NONE, PRIVATE|ANON|NORESERVE
            assert base not in (None, C.c_void_p(-1).value)
            self.base = base
            self.fds = {}
            for ci in [self.body] + self.hot:
                fd = os.memfd_create("fsk-long-row-%d" % ci)
                os.ftruncate(fd, CHUNK)
                self.fds[ci] = fd
            for ci in range(nchunks):
                fd = self.fds.get(ci, self.fds[self.body])
                a = libc.mmap(base + ci * CHUNK, CHUNK, 0x1 | 0x2, 0x01 | 0x10, fd, 0)    # RW, SHARED|FIXED
                assert a == base + ci * CHUNK, C.get_errno()
            return
        t = torch()
        t.zeros(1, device=dev())                      # the primary context, current on this thread
        d = self.drv = _Driver()
        cu = d.cu
        prop = d.prop(d.device())
        gran = C.c_size_t()
        d.ok(cu.cuMemGetAllocationGranularity(C.byref(gran), prop, 0), "cuMemGetAllocationGranularity")
        assert CHUNK % gran.value == 0, gran.value
        ptr = C.c_uint64()
        d.ok(cu.cuMemAddressReserve(C.byref(ptr), C.c_size_t(self.nbytes), C.c_size_t(0), C.c_uint64(0),
                                    C.c_uint64(0)), "cuMemAddressReserve")
        self.base = ptr.value
        self.handles = {}
        for ci in [self.body] + self.hot:
            h = C.c_uint64()
            d.ok(cu.cuMemCreate(C.byref(h), C.c_size_t(CHUNK), prop, C.c_uint64(0)), "cuMemCreate")
            self.handles[ci] = h.value
        self.mapped = []
        for ci in range(nchunks):
            h = self.handles.get(ci, self.handles[self.body])
            d.ok(cu.cuMemMap(C.c_uint64(self.base + ci * CHUNK), C.c_size_t(CHUNK), C.c_size_t(0), C.c_uint64(h),
                             C.c_uint64(0)), "cuMemMap")
            self.mapped.append(ci)
        desc = (C.c_int * 3)(1, d.device(), 3)         # location (DEVICE, dev), PROT_READWRITE
        d.ok(cu.cuMemSetAccess(C.c_uint64(self.base), C.c_size_t(self.nbytes), desc, C.c_size_t(1)),
             "cuMemSetAccess")

    def write(self, e0, a):
        t = torch()
        self.flat[e0:e0 + a.size] = upload(np.ascontiguousarray(a))
        sync()

    def read(self, e0, e1):
        return self.flat[e0:e1].cpu().numpy().copy()

    def is_hot(self, e0, e1):
        return all(ci in self.hot for ci in range(e0 * self.es // CHUNK, (e1 - 1) * self.es // CHUNK + 1))

    def close(self):
        self.t = self.flat = None
        if self.emu:
            assert self.libc.munmap(C.c_void_p(self.base), C.c_size_t(self.nbytes)) == 0
            for fd in self.fds.values():
                os.close(fd)
            return
        sync()
        cu = self.drv.cu
        for ci in self.mapped:
            self.drv.ok(cu.cuMemUnmap(C.c_uint64(self.base + ci * CHUNK), C.c_size_t(CHUNK)), "cuMemUnmap")
        self.drv.ok(cu.cuMemAddressFree(C.c_uint64(self.base), C.c_size_t(self.nbytes)), "cuMemAddressFree")
        for h in self.handles.values():
            self.drv.ok(cu.cuMemRelease(C.c_uint64(h)), "cuMemRelease")


def loud(rng, n, dtype, rate=48000):
    """noise of sigma 0.4 plus a 0.4 tone at 1700 Hz (inside the Bell202 and Bell103 bands)"""
    x = 0.4 * rng.standard_normal(n) + 0.4 * np.sin(2 * np.pi * 1700.0 / rate * np.arange(n))
    x = x.astype(np.float32)
    return pcm(x) if np.dtype(dtype) == np.int16 else x


_ROWS = {}


@pytest.fixture(scope="module")
def rows():
    """the aliased layouts, one per sample type, made on first use and unmapped at the end of the module"""
    info = {}
    if not emulated():
        torch().zeros(1, device=dev())             # the primary context, current on this thread
        torch().cuda.empty_cache()
        info["before"] = _Driver().mem_info()[0]

    def get(dtype):
        k = np.dtype(dtype).str
        if k not in _ROWS:
            _ROWS[k] = AliasedRows(dtype)
        return _ROWS[k]
    yield get
    phys = sum(r.physical for r in _ROWS.values())
    for r in list(_ROWS.values()):
        r.close()
    _ROWS.clear()
    assert phys <= 128 << 20, phys
    if not emulated():
        torch().cuda.empty_cache()
        after = _Driver().mem_info()[0]
        print("long rows: %d MB physical; cuMemGetInfo free %d MB before, %d MB after"
              % (phys >> 20, info["before"] >> 20, after >> 20))


# ---------------------------------------------------------------------------------------------------
# families and streams
# ---------------------------------------------------------------------------------------------------
FAMS = list(rxfam.FAMILIES)


def preset_of(fam):
    """(preset, number of words) of a family's stream: the generic kernel's bit periods need 25 baud"""
    if fam.startswith("generic"):
        return ("25", 48000), 3
    return (("300", 48000) if fam.startswith("prefix-table") else ("1200", 48000)), 12


_STREAMS = {}


def stream(preset, nwords):
    """nwords random words from the oracle's transmitter at amplitude 0.7, sigma = 0.01 noise"""
    key = (preset, nwords)
    if key not in _STREAMS:
        m = orc.Mode(preset[0], sample_rate=preset[1])
        rng = np.random.default_rng(7 + nwords + int(preset[0]))
        words = rng.integers(0, 1 << m.n_data_bits, nwords, dtype=np.uint64).astype(np.uint32)
        x = orc.tx_words(m, words, 0.7, 4096, True)
        x = (x + np.float32(0.01) * rng.standard_normal(x.size).astype(np.float32)).astype(np.float32)
        _STREAMS[key] = (m, x)
    return _STREAMS[key]


def decode(eng, fam, x, n, pos, nrows=1, row=0):
    """one call over the [nrows, stride] tensor x (row `row` starts at pos; the others are done) ->
    (records of that row's stream(s) as bytes, then the auto states of the row, and states as numpy)"""
    f = rxfam.FAMILIES[fam]
    k = f.get("k", 1)
    st = np.zeros(nrows * k, mm.STATE_DTYPE)
    st["done"] = 1
    st["pos"][row * k:(row + 1) * k] = pos
    st["done"][row * k:(row + 1) * k] = 0
    bands = None
    if f["call"] == "tones":
        p = eng.params
        pairs = [mm.tone_bands(p, 1200.0, 2200.0) if preset_of(fam)[0][0] == "1200" else mm.tone_bands(p, 1270.0, 1070.0)]
        pairs += [mm.tone_bands(p, 1070.0, 1270.0), [p.nbands, p.nbands]][:k - 1]
        bands = np.array(pairs * nrows, np.int32).reshape(nrows * k, 2)
    r = rxfam.call(eng, fam, x, n=n, bands=bands, states=st, max_frames=96, rec_band=True)
    rxfam.check_family(fam, r.k)
    recs = r.recs[row * k:(row + 1) * k]
    if r.auto is not None:
        recs.append(r.auto.cpu().numpy()[row].tobytes())
    return recs, r.st[row * k:(row + 1) * k].copy()


def placement(case, n, spb, xlen):
    """(P = first sample of the stream, start = the state's pos) for a row of n samples"""
    if case == "cut":
        P = n - xlen + int(spb * 5)     # the last frame runs half a frame past n
    else:
        P = n - xlen
    start = P - int(spb * 31) if case == "earlier" else P
    return P, start


def small_twin(big, n, P, start, x, src):
    """the same samples in a small row at base p0 = start mod 128, loud noise after its own n; -> (tensor, n, p0)"""
    p0 = start % 128
    lead = big.read(start - p0, P)
    body = x if src == "f32" else pcm(x)
    seg = np.concatenate([lead, body]).astype(big.dtype)
    ns = p0 + (n - start)
    tail = loud(np.random.default_rng(5), 8192, big.dtype)
    row = np.concatenate([seg[:ns], seg[ns:], tail[:8192 - (seg.size - ns)]])
    stride = (row.size + 7) & ~7
    buf = np.zeros((1, stride), big.dtype)
    buf[0, :row.size] = row
    buf[0, row.size:] = tail[:stride - row.size]
    return upload(buf), ns, p0


def check_equal(big_run, small_run, shift, what):
    (rb, sb), (rs, ss) = big_run, small_run
    assert len(rb) == len(rs)
    for i, (a, b) in enumerate(zip(rb, rs)):
        assert a == b, (what, "records" if i < len(sb) else "auto state", i, len(a) // 20, len(b) // 20,
                        first_diff(a, b))
    sb = sb.copy()
    assert (sb["pos"] - ss["pos"] == shift).all(), (what, sb["pos"], ss["pos"], shift)
    sb["pos"] = ss["pos"]
    assert sb.tobytes() == ss.tobytes(), (what, sb, ss)


def first_diff(a, b):
    fa, fb = np.frombuffer(a, mm.FRAME_DTYPE), np.frombuffer(b, mm.FRAME_DTYPE)
    for i in range(min(fa.size, fb.size)):
        if fa[i].tobytes() != fb[i].tobytes():
            return "record %d of %d/%d: %r vs %r" % (i, fa.size, fb.size, fa[i], fb[i])
    return "lengths %d/%d" % (fa.size, fb.size)


def run_case(rows, monkeypatch, fam, n, case, row=0):
    src = rxfam.FAMILIES[fam]["src"]
    preset, nwords = preset_of(fam)
    m, x = stream(preset, nwords)
    spb = float(m.derived().nsamples_per_bit)
    big = rows(np.float32 if src == "f32" else np.int16)
    P, start = placement(case, n, spb, x.size)
    e0 = row * STRIDE
    assert big.is_hot(e0 + start - 128, e0 + P + x.size + 1), (n, case)
    big.write(e0 + P, x if src == "f32" else pcm(x))
    eng = rxfam.new_engine(monkeypatch, fam, lambda: mm.RxEngine.for_mode(*preset))
    nrows = 2 if row else 1
    got = decode(eng, fam, big.t[:nrows], n, start, nrows=nrows, row=row)
    xs, ns, p0 = small_twin(big, e0 + n, e0 + P, e0 + start, x, src)
    want = decode(eng, fam, xs, ns, p0)
    what = "%s n=%d (2^32 - %d) %s" % (fam, n, TOP - n, case)
    check_equal(got, want, start - p0, what)
    st = want[1]
    assert (st["done"][:2] == 1).all(), what          # (channels-3: the third channel is disabled)
    if case == "at-start" and not fam.startswith("generic"):
        assert st["nframes"][0] >= nwords - 1, (what, st["nframes"])
    return want, xs, ns, p0, m


# ---------------------------------------------------------------------------------------------------
# the tests
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("nid,n", ROW_LENGTHS, ids=[i for i, _ in ROW_LENGTHS])
@pytest.mark.parametrize("fam", FAMS)
def test_stream_at_the_end_of_a_long_row(rows, monkeypatch, fam, nid, n, case):
    """A stream at the end of a row of n samples decodes as at the start of a small row."""
    rxfam.skip_tma(fam)
    run_case(rows, monkeypatch, fam, n, case)


@pytest.mark.parametrize("fam", FAMS)
def test_second_row_beyond_2_32_elements(rows, monkeypatch, fam):
    """Row 1 of two rows of 2^32 samples starts at element 2^32: the row offsets are size_t."""
    rxfam.skip_tma(fam)
    run_case(rows, monkeypatch, fam, MAX_ROW, "at-start", row=1)


def test_small_row_is_the_oracles(rows, monkeypatch):
    """The small twin of the per-candidate float case against the screened oracle: the comparison above is
    anchored to what the reference decodes from these samples."""
    (recs, st), xs, ns, p0, m = run_case(rows, monkeypatch, "per-candidate", MAX_ROW, "at-start")
    seg = xs.cpu().numpy()[0, p0:ns].astype(np.float32)
    want, robust = tie_screen.screen(m, seg)
    assert robust
    got = np.frombuffer(recs[0], mm.FRAME_DTYPE)
    compare_frames(as_oracle_frames(got), want["frames"], "small twin")
    compare_reports(reports_of(got, st[0]), want["reports"], "small twin")


@pytest.mark.parametrize("nid,n", [ROW_LENGTHS[0], ROW_LENGTHS[-3]], ids=[ROW_LENGTHS[0][0], ROW_LENGTHS[-3][0]])
def test_find_frame_and_detect_carrier_near_2_32(rows, nid, n):
    """fsk_b200_find_frame_batch with offset[s] and nvalid[s] near 2^32 (the search window running past
    nvalid), and fsk_b200_detect_carrier_batch with offset[s] near 2^32, against the same samples in a
    small row."""
    t = torch()
    m, x = stream(("1200", 48000), 12)
    big = rows(np.float32)
    P = n - x.size
    big.write(P, x)
    eng = mm.RxEngine.for_mode("1200", 48000)
    p = eng.params
    spb = int(m.derived().nsamples_per_bit)
    offs = np.array([P + 3, P + 40 * spb + 1, n - 6 * spb, n - 2 * spb, n - 1], np.int64)
    xs, ns, p0 = small_twin(big, n, P, P, x, "f32")

    def ff(buf, base, nvalid):
        k = offs.size
        u = lambda a: upload(np.asarray(a, np.uint32).view(np.int32))
        o = u(offs - base)
        fr = []
        for i in range(k):
            f = eng.find_frame_batch(buf, u([nvalid]), u([0]), u([p.try_max_nocarrier]), u([max(1, p.try_max_nocarrier // 3)]),
                                     upload(np.array([np.inf], np.float32)),
                                     offset=o[i:i + 1], expect_sel=upload(np.array([1], np.uint8)))
            sync()
            assert eng.last_kernel().startswith("k_find_frame"), eng.last_kernel()
            fr.append(f.cpu().numpy().tobytes())
        return fr
    a = ff(big.t[:1], 0, n)
    b = ff(xs, P - p0, ns)
    assert a == b
    assert any(np.frombuffer(r, mm.FRAME_DTYPE)["confidence"][0] > 0 for r in a)
    fft = int(p.fftsize)
    for off in (P + 100, n - fft):
        o1 = upload(np.array([off], np.uint32).view(np.int32))
        o2 = upload(np.array([off - (P - p0)], np.uint32).view(np.int32))
        g = mm.detect_carrier_batch(fft, big.t[:1], fft, 0.001, offset=o1).cpu().numpy()
        w = mm.detect_carrier_batch(fft, xs, fft, 0.001, offset=o2).cpu().numpy()
        assert (g == w).all() and int(w[0]) > 0, (off, g, w)


def test_rx_calls_refuse_rows_above_the_limit():
    """nsamples_all > 2^32 - 4 returns -EINVAL in every rx call and launches nothing; 2^32 - 4 is taken."""
    t = torch()
    eng = mm.RxEngine.for_mode("1200", 48000)
    lib = mm.api.lib()
    x = t.zeros((1, 64), dtype=t.float32, device=dev())
    x16 = t.zeros((1, 64), dtype=t.int16, device=dev())
    fr = t.zeros((1, 4, 5), dtype=t.int32, device=dev())
    st = t.zeros((1, mm.STATE_WORDS), dtype=t.int32, device=dev())
    ast = t.zeros((1, mm.api.AUTO_STATE_BYTES), dtype=t.uint8, device=dev())
    each = upload(np.array([64], np.int32))
    tb = eng.tone_bands(1200.0, 2200.0, device=dev())
    eng.set_auto_carrier(autoorc.DEFAULT_THRESHOLD)
    P = mm.api._ptr
    h = mm.api._stream_handle()
    calls = {
        "rx_batch": lambda n: lib.fsk_b200_rx_batch(eng._e, P(x), 1, 1 << 40, P(each), n, P(fr), 4, P(st), h),
        "rx_batch_s16": lambda n: lib.fsk_b200_rx_batch_s16(eng._e, P(x16), 1, 1 << 40, P(each), n, P(fr), 4, P(st), h),
        "rx_batch_auto": lambda n: lib.fsk_b200_rx_batch_auto(eng._e, P(x), 1, 1 << 40, P(each), n, P(fr), 4, P(st),
                                                              P(ast), None, h),
        "rx_batch_auto_s16": lambda n: lib.fsk_b200_rx_batch_auto_s16(eng._e, P(x16), 1, 1 << 40, P(each), n, P(fr), 4,
                                                                      P(st), P(ast), None, h),
        "rx_batch_tones": lambda n: lib.fsk_b200_rx_batch_tones(eng._e, P(x), 1, 1 << 40, P(each), n, P(tb), P(fr), 4,
                                                                P(st), h),
        "rx_batch_tones_s16": lambda n: lib.fsk_b200_rx_batch_tones_s16(eng._e, P(x16), 1, 1 << 40, P(each), n, P(tb),
                                                                        P(fr), 4, P(st), h),
        "rx_batch_channels": lambda n: lib.fsk_b200_rx_batch_channels(eng._e, P(x), 1, 1 << 40, P(each), n, 1, P(tb),
                                                                      P(fr), 4, P(st), h),
        "rx_batch_channels_s16": lambda n: lib.fsk_b200_rx_batch_channels_s16(eng._e, P(x16), 1, 1 << 40, P(each), n, 1,
                                                                              P(tb), P(fr), 4, P(st), h),
    }
    for name, call in calls.items():
        for n in (TOP - 3, TOP - 1):
            before = mm.launch_count()
            assert call(n) == -22, (name, n)
            assert mm.launch_count() == before, (name, n)
            assert "2^32 - 4" in mm.api.lib().fsk_b200_last_error().decode(), name
        before = mm.launch_count()
        assert call(MAX_ROW) == 0, name         # per-row lengths (64) bound the rows
        sync()
        assert mm.launch_count() > before, name
    hf = np.zeros((1, 4), mm.FRAME_DTYPE)
    hs = np.zeros(1, mm.STATE_DTYPE)
    for name, fn, buf in (("rx_batch_host", lib.fsk_b200_rx_batch_host, np.zeros((1, 64), np.float32)),
                          ("rx_batch_host_s16", lib.fsk_b200_rx_batch_host_s16, np.zeros((1, 64), np.int16))):
        before = mm.launch_count()
        assert fn(eng._e, buf.ctypes.data_as(C.c_void_p), 1, 1 << 40, TOP - 1, hf.ctypes.data_as(C.c_void_p), 4,
                  hs.ctypes.data_as(C.c_void_p)) == -22, name
        assert mm.launch_count() == before, name


@pytest.mark.parametrize("start", [10, 0])
def test_stream_push_caps_a_row_at_the_limit(rows, start):
    """The live push with pos = 0 (no tail move) and a row `start` samples short of 2^32 - 4: what fits
    below the limit is appended, the rest counted in `dropped`, and nothing at or past 2^32 - 4 changes."""
    t = torch()
    big = rows(np.float32)
    have = MAX_ROW - start
    before = big.read(have - 64, MAX_ROW + 64)
    chunk = np.arange(1, 33, dtype=np.float32)[None, :] * np.float32(0.25)
    fill = upload(np.array([have], np.uint32).view(np.int32))
    dropped = t.zeros(1, dtype=t.int32, device=dev())
    st = t.zeros((1, mm.STATE_WORDS), dtype=t.int32, device=dev())
    mm.stream_push(big.t[:1], fill, st, upload(chunk), dropped=dropped)
    sync()
    f = int(fill.cpu().numpy().view(np.uint32)[0])
    d = int(dropped.cpu().numpy()[0])
    assert (f, d) == (MAX_ROW, 32 - start), (f, d)
    after = big.read(have - 64, MAX_ROW + 64)
    want = before.copy()
    want[64:64 + start] = chunk[0, :start]
    assert after.tobytes() == want.tobytes()
    big.write(have - 64, before)
    sn = mm.states_to_numpy(st)
    assert int(sn["pos"][0]) == 0 and int(sn["nframes"][0]) == 0


def test_no_mapping_is_left_behind():
    """A layout made and unmapped returns its memory: the reserved range is gone and free memory is back."""
    if emulated():
        r = AliasedRows(np.int16, rows=1)
        base, nb = r.base, r.nbytes
        r.close()
        with open("/proc/self/maps") as fh:
            for line in fh:
                lo, hi = (int(v, 16) for v in line.split()[0].split("-"))
                assert hi <= base or lo >= base + nb, line
        return
    t = torch()
    t.cuda.empty_cache()
    drv = _Driver()
    t.zeros(1, device=dev())
    free0 = drv.mem_info()[0]
    r = AliasedRows(np.int16, rows=1)
    t.cuda.empty_cache()
    free1 = drv.mem_info()[0]
    base, phys = r.base, r.physical
    r.close()
    t.cuda.empty_cache()
    free2 = drv.mem_info()[0]
    print("aliased int16 row: %d MB physical; free %d -> %d -> %d MB" % (phys >> 20, free0 >> 20, free1 >> 20,
                                                                       free2 >> 20))
    assert free0 - free1 >= phys - (8 << 20)
    assert abs(free2 - free0) <= 8 << 20, (free0, free2)
    pb, ps = C.c_uint64(), C.c_size_t()
    assert drv.cu.cuMemGetAddressRange_v2(C.byref(pb), C.byref(ps), C.c_uint64(base)) != 0


# ---------------------------------------------------------------------------------------------------
# transmitter: lead-ins and lengths at 2^32 - 1
# ---------------------------------------------------------------------------------------------------
def test_tx_channel_lead_in_near_2_32():
    """A channel whose lead-in alone passes a small nsamples_out adds nothing to its row; out_len is the
    lead-in plus the signal, saturated at 2^32 - 1."""
    t = torch()
    eng = mm.TxEngine.for_mode("1200", 48000, float_samples=True)
    text = upload(np.frombuffer(b"HELLO 2^32", np.uint8).reshape(1, -1).repeat(3, 0).copy())
    lens = upload(np.array([10, 10, 10], np.int32))
    tones = eng.tone_pairs([1200.0, 1070.0, 2025.0], [2200.0, 1270.0, 2225.0], device=dev())
    leads = np.array([0, TOP - 1, TOP - 4000], np.uint32)
    lead = upload(leads.view(np.int32))
    out = t.full((1, 4096), 7.0, dtype=t.float32, device=dev())
    r = eng.text_channels(text, lens, tones, 3, 4000, lead_in=lead, out=out)
    o, out_len = r[0], r[1]
    sync()
    ref = t.full((1, 4096), 7.0, dtype=t.float32, device=dev())
    r1 = eng.text_channels(text[:1], lens[:1], tones[:1], 1, 4000, lead_in=lead[:1], out=ref)
    sync()
    assert o.cpu().numpy().tobytes() == r1[0].cpu().numpy().tobytes()
    ol = out_len.cpu().numpy().view(np.uint32)
    sig = int(r1[1].cpu().numpy().view(np.uint32)[0])
    assert sig > 0 and ol[0] == sig
    assert ol[1] == TOP - 1 and ol[2] == min(TOP - 1, TOP - 4000 + sig), (ol, sig)


def test_tx_channels_length_bound_at_2_32():
    """The longest channel a text_stride allows plus nsamples_out may reach 2^32 - 1 samples, not 2^32."""
    t = torch()
    eng = mm.TxEngine.for_mode("1200", 48000, float_samples=True)
    need = lambda S: mm.tx_max_samples(eng, S, mm.api.TX_FINAL)
    lo, hi = 1, 1 << 24                     # the largest text_stride whose channel fits below 2^32 - 1 - 64
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if 0 < need(mid) <= TOP - 1 - 64 else (lo, mid)
    S = lo
    nout = TOP - 1 - need(S)
    assert 64 <= nout < 4096, (S, need(S))
    text = t.zeros((1, S), dtype=t.uint8, device=dev())
    text[0, 0] = ord("A")
    lens = upload(np.array([1], np.int32))
    tones = eng.tone_pairs([1200.0], [2200.0], device=dev())
    out = t.zeros((1, 4096), dtype=t.float32, device=dev())
    out_len = t.zeros(1, dtype=t.int32, device=dev())
    lib, P = mm.api.lib(), mm.api._ptr
    call = lambda n: lib.fsk_b200_tx_text_channels(eng._te, P(text), 1, 1, S, P(lens), P(tones), None, P(out), 4096,
                                                   n, P(out_len), mm.api._stream_handle())
    before = mm.launch_count()
    assert call(nout + 1) == -22
    assert mm.launch_count() == before
    assert call(nout) == 0
    sync()
    assert mm.launch_count() > before
    assert int(out_len.cpu().numpy()[0]) > 0 and bool((out.cpu().numpy()[0, :64] != 0).any())
