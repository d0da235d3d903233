"""-M / -S per stream: fsk_b200_rx_batch_tones / _s16 (the per-candidate rx kernel with a tone table per
stream, AUTO = 2) against the reference's own vectors, the FLAT oracle and the fixed-tone engine.

Stream s of a call must behave like the reference CLI run on that row with -M f_mark[s] -S f_space[s]:
the records and states of fsk_b200_rx_batch on an engine built for that pair.  The per-stream tables are
filled from the unit-circle table whose entries are bit-identical to a fixed-tone engine's, so on the
engine's own pair the records equal the forced per-candidate rx_batch bit for bit.  Random pairs are
screened with tests/tie_screen.py first: robust streams must give the oracle's records exactly, the
others the same frame count within one.

The CPU tests pin fsk_b200_tone_bands to fsk_b200_rx_params_derive and run the `gpu` tests of this file
on the host SIMT emulation of the kernels (tests/emu)."""
import ctypes as C
import zlib

import numpy as np
import pytest

import golden_util as gu
import orc
import refcases
import tie_screen
from gpudev import dev, mm, pcm, rows, state_rows, sync, torch, upload
from rxcases import (ANSWER, COVER, KEYS, ORIGINATE, TONE_PRESETS, auto_combos, duplex_case, lay_out, on_pair,
                     random_pair, transmission)
from rxfam import as_oracle_frames, check_against_oracle, compare_frames, reports_of

EINVAL, ENOTSUP = 22, 95
f32 = np.float32


# --------------------------------------------------------------------------
# CPU: the band arithmetic, the cover table, the emulated kernels
# --------------------------------------------------------------------------
def derive_bands(cfg):
    """(rc, b_mark, b_space) of fsk_b200_rx_params_derive on this config"""
    p = mm().RxParams()
    rc = mm().lib().fsk_b200_rx_params_derive(C.byref(cfg), C.byref(p))
    return rc, int(p.b_mark), int(p.b_space)


def helper(params, fm, fs):
    b = (C.c_uint32 * 2)()
    rc = mm().lib().fsk_b200_tone_bands(C.byref(params), f32(fm), f32(fs), b)
    return rc, int(b[0]), int(b[1])


def test_tone_bands_equal_the_derived_bands():
    """fsk_b200_tone_bands against fsk_b200_rx_params_derive (fsk_plan_new's arithmetic) on random modes,
    sample rates, -b values and tones, a third of them within a float ulp of a band edge: the same bands,
    and -EINVAL exactly where the derivation fails."""
    rng = np.random.default_rng(20261016)
    ndraw = nfail = nedge = 0
    for _ in range(3000):
        mode = TONE_PRESETS[int(rng.integers(len(TONE_PRESETS)))]
        rate = float([8000, 11025, 22050, 44100, 48000, int(rng.integers(4000, 96001))][int(rng.integers(6))])
        bw = 0.0 if rng.random() < 0.4 else float(f32(rng.choice([rng.uniform(1, 400), rng.integers(1, 400)])))
        base = mm().rx_config_for_mode(mode, rate, band_width=bw)
        params = mm().RxParams()
        if mm().lib().fsk_b200_rx_params_derive(C.byref(base), C.byref(params)) != 0:
            continue
        w, nb = f32(params.band_width), int(params.nbands)
        tones = []
        for _t in range(2):
            u = rng.random()
            if u < 0.35:                        # within a few ulps of a band edge: (f + bw/2) / bw ~ k
                k = int(rng.integers(1, nb + 2))
                f = f32(f32(k) * w - w / f32(2))
                for _s in range(int(rng.integers(-3, 4))):
                    f = np.nextafter(f, f32(np.inf) if _s >= 0 else f32(0), dtype=f32)
                tones.append(f)
                nedge += 1
            elif u < 0.5:                       # beyond the last band
                tones.append(f32(rng.uniform(nb - 1, 2 * nb + 2) * w))
            else:
                tones.append(f32(rng.uniform(0.01, nb) * w))
        fm, fs = tones
        if fm <= 0 or fs <= 0:                  # 0 means "the preset's tone" to rx_config_for_mode
            continue
        cfg = mm().rx_config_for_mode(mode, rate, band_width=bw, f_mark=float(fm), f_space=float(fs))
        assert f32(cfg.band_width) == w
        rc, bm, bs = derive_bands(cfg)
        hrc, hm, hs = helper(params, cfg.f_mark, cfg.f_space)
        ndraw += 1
        if rc != 0:
            nfail += 1
            assert hrc == -EINVAL, (mode, rate, bw, cfg.f_mark, cfg.f_space)
        else:
            assert hrc == 0 and (hm, hs) == (bm, bs), (mode, rate, bw, cfg.f_mark, cfg.f_space, (hm, hs), (bm, bs))
        # the Python form goes through the same helper
        if hrc == 0:
            assert mm().tone_bands(params, cfg.f_mark, cfg.f_space) == (hm, hs)
        else:
            with pytest.raises(ValueError):
                mm().tone_bands(params, cfg.f_mark, cfg.f_space)
    assert ndraw > 2000 and 200 < nfail < ndraw - 1000 and nedge > 1000, (ndraw, nfail, nedge)


def test_tone_bands_reject_negative_and_non_finite_tones():
    params = mm().rx_params(mm().rx_config_for_mode("1200", 48000))
    assert helper(params, 1200.0, 2200.0) == (0, 6, 11)
    assert helper(params, 0.0, 2200.0) == (0, 0, 11)
    for bad in (-1.0, -1e-3, -np.inf, np.inf, np.nan):
        assert helper(params, bad, 2200.0)[0] == -EINVAL, bad
        assert helper(params, 1200.0, bad)[0] == -EINVAL, bad
    assert mm().lib().fsk_b200_tone_bands(C.byref(params), f32(1200), f32(2200), None) == -EINVAL


def test_the_cover_table_is_the_auto_combo_list():
    assert set(COVER) == auto_combos()


def test_live_receiver_refuses_tones_with_auto_carrier():
    from minimodem_b200.serving import LiveReceiver
    with pytest.raises(ValueError, match="exclude"):
        LiveReceiver("1200", 48000, 2, auto_carrier=0.001, tones=np.zeros((2, 2), np.int32))


def test_gpu_stream_tones_file_on_the_emulated_kernels():
    """The `gpu` tests below on the host SIMT emulation of the kernels: copies landing late, the
    approximate units moved by up to 64 ulp."""
    from gpudev import run_emulated
    tail = run_emulated("gpu", "late", 2400, module="test_gpu_stream_tones.py",
                        extra_env={"FSK_EMU_ULP": "64"})
    assert " passed" in tail and "failed" not in tail


def test_reference_vectors_on_the_emulated_kernels_eager_copies():
    from gpudev import run_emulated
    tail = run_emulated("reference_vectors", "eager", 900, module="test_gpu_stream_tones.py")
    assert " passed" in tail and "failed" not in tail


# --------------------------------------------------------------------------
# streams
# --------------------------------------------------------------------------


_CASES = {}


def random_case(mode, rate):
    """3..8 streams of one mode, each on its own random pair, with ragged lead-ins and noise; stream 0 is cut
    mid-frame (its row holds more than its length).  Returns (engine params of the preset, marks, spaces,
    streams, lengths, [(oracle result, robust)])."""
    key = (mode, rate)
    if key in _CASES:
        return _CASES[key]
    rng = np.random.default_rng(zlib.crc32(repr(key).encode()))
    base = orc.Mode(mode, sample_rate=rate)
    bw = float(base.band_width)
    nbands = int((rate + bw / 2) / bw) // 2 + 1
    marks, spaces, streams, lens, screened = [], [], [], [], []
    for s in range(int(rng.integers(3, 9))):
        fm, fs = random_pair(rng, bw, nbands)
        m = on_pair(mode, rate, fm, fs)
        audio = transmission(rng, m, int(rng.integers(4, 8)), float(rng.uniform(0.3, 1.0)))
        x, lead = lay_out(rng, m, audio, rng.uniform(1e-4, 3e-3))
        n = x.size if s else lead + int(audio.size * rng.uniform(0.5, 0.8))
        marks.append(fm)
        spaces.append(fs)
        streams.append(x)
        lens.append(n)
        screened.append(tie_screen.screen(m, x[:n]))
    _CASES[key] = (marks, spaces, streams, np.array(lens, np.int32), screened)
    return _CASES[key]


def run_tones(eng, buf, n, lens, bands, states=None, max_frames=None):
    t = torch()
    frames, st = eng.rx_batch_tones(upload(buf), bands, nsamples=n,
                                    nsamples_each=upload(np.asarray(lens, np.int32)),
                                    states=states, max_frames=max_frames)
    sync()
    return frames, st


# --------------------------------------------------------------------------
# the reference CLI's own vectors, each on its own pair, in one call
# --------------------------------------------------------------------------
VECTORS = ["small-1200", "opt-mark-space", "opt-inverted", "small-1200-float-noise", "more-quiet-noise"]


def vector_audio(name):
    case = refcases.BY_NAME[name]
    g = gu.load(name)
    a = gu.audio(case, g)
    if case["rxnoise"]:             # --Xrxnoise, as tests/test_gpu_parity.py applies it
        a = (a + np.float32(-0.5) * np.float32(np.float32(case["rxnoise"]) * 2)).astype(np.float32)
    return case, g, a


@pytest.mark.gpu
def test_reference_vectors_each_on_its_own_pair_in_one_call():
    """One rx_batch_tones call on a "1200" @ 48 kHz engine decodes the committed audio of five reference
    runs, each on the -M / -S of its own command line (opt-inverted as the preset pair with inverted=True):
    every row prints the reference's stdout byte for byte and its NOCARRIER lines.  The three int16 vectors
    once more as int16 rows give the same records, bit for bit."""
    t = torch()
    eng = mm().RxEngine.for_mode("1200", 48000)
    audio, marks, spaces, inv = [], [], [], []
    for name in VECTORS:
        case, g, a = vector_audio(name)
        _, rx = gu.modes(case)
        audio.append(a)
        inverted = bool(case["rx_mkw"].get("inverted", False))
        pre = orc.Mode("1200", mark=case["rx_mkw"].get("mark", 0.0), space=case["rx_mkw"].get("space", 0.0))
        marks.append(float(pre.mark_f))
        spaces.append(float(pre.space_f))
        inv.append(inverted)
        assert (float(rx.mark_f), float(rx.space_f)) == ((spaces[-1], marks[-1]) if inverted else (marks[-1], spaces[-1]))
    bands = eng.tone_bands(marks, spaces, inverted=inv, device=dev())
    assert bands.cpu().numpy().tolist() == [[6, 11], [8, 11], [11, 6], [6, 11], [6, 11]]
    buf, n = rows(audio, np.float32, 4)
    lens = np.array([a.size for a in audio], np.int32)
    frames, states = run_tones(eng, buf, n, lens, bands)
    assert eng.last_kernel().startswith("k_rx_tones<G=8,W=3,L=2,mode=0(per-candidate),fill=0,src=f32")
    kind = mm().decoder_for_mode("1200", 8)
    out, cnt = eng.decode_batch(kind, frames, states)
    sync()
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    fr, st = mm().frames_to_numpy(frames), mm().states_to_numpy(states)
    assert (st["done"] == 1).all()
    for s, name in enumerate(VECTORS):
        case, g, _ = vector_audio(name)
        _, rx = gu.modes(case)
        assert out[s, :cnt[s]].tobytes() == bytes(g["stdout"]), name
        lines = [orc.report_line(rx, r) for r in reports_of(fr[s, :int(st["nframes"][s])], st[s])]
        want = gu.stat_lines(g)
        assert len(lines) >= len(want) >= 1, (name, lines, want)
        for x, y in zip(lines, want):
            fa, fb = x.split(), y.split()
            assert fa[:3] == fb[:3] and fa[4:] == fb[4:], (name, x, y)
            assert gu.close(float(fa[3].split("=")[1]), float(fb[3].split("=")[1]), 2e-3, cond=gu.CONF_COND)
    s16 = [i for i, name in enumerate(VECTORS) if "audio_s16" in gu.load(name).files]
    assert len(s16) == 3
    b16, n16 = rows([gu.load(VECTORS[i])["audio_s16"] for i in s16], np.int16, 8)
    f16, st16 = run_tones(eng, b16, n16, lens[s16], bands[t.tensor(s16, device=bands.device)].contiguous())
    assert "src=s16" in eng.last_kernel()
    f16, st16 = mm().frames_to_numpy(f16), mm().states_to_numpy(st16)
    for j, i in enumerate(s16):
        k = int(st["nframes"][i])
        assert int(st16["nframes"][j]) == k and f16[j, :k].tobytes() == fr[i, :k].tobytes(), VECTORS[i]


# --------------------------------------------------------------------------
# every instance, random pairs
# --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("key", KEYS, ids=[str(k) for k in KEYS])
def test_every_instance_on_random_pairs(key):
    """Every AUTO_COMBOS shape, float and int16: each stream on its own pair gives the FLAT oracle's records
    on that pair; int16 rows give the float rows' records and states bit for bit, in one pass and resumed
    at position 13."""
    mode, rate = COVER[key]
    marks, spaces, streams, lens, screened = random_case(mode, rate)
    eng = mm().RxEngine.for_mode(mode, rate)
    bands = eng.tone_bands(marks, spaces, device=dev())
    b = bands.cpu().numpy()
    assert (b[:, 0] != b[:, 1]).all() and (b[:, 0] > b[:, 1]).any() and (b[:, 0] < b[:, 1]).any()
    buf, n = rows(streams, np.float32, 4)
    frames, states = run_tones(eng, buf, n, lens, bands)
    G, W, L = key
    assert eng.last_kernel().startswith("k_rx_tones<G=%d,W=%d,L=%d,mode=0(per-candidate),fill=0,src=f32" % (G, W, L))
    st = mm().states_to_numpy(states)
    assert (st["done"] == 1).all()
    check_against_oracle(screened, mm().frames_to_numpy(frames), st, str(key))
    p16 = [pcm(a) for a in streams]
    b16, _ = rows(p16, np.int16, 8)
    b32, _ = rows([a.astype(np.float32) * np.float32(1.0 / 32768.0) for a in p16], np.float32, 8)
    for resume in (0, 13):
        outs = []
        for bb in (b32, b16):
            st0 = np.zeros(len(streams), mm().STATE_DTYPE)
            st0["pos"][:] = resume
            outs.append(run_tones(eng, bb, n, lens, bands, states=state_rows(st0)))
            assert eng.last_kernel().startswith("k_rx_tones<G=%d,W=%d,L=%d," % (G, W, L))
        assert "src=s16" in eng.last_kernel()
        (fa, sa), (fb, sb) = outs
        sa, sb = mm().states_to_numpy(sa), mm().states_to_numpy(sb)
        assert sa.tobytes() == sb.tobytes(), (key, resume)
        fa, fb = mm().frames_to_numpy(fa), mm().frames_to_numpy(fb)
        for s in range(len(streams)):
            k = int(sa["nframes"][s])
            assert fa[s, :k].tobytes() == fb[s, :k].tobytes(), (key, s, resume)
        assert sa["nframes"].sum() >= len(streams)


def preset_streams(mode, rate, count, seed):
    """streams on the preset's own tones, ragged lead-ins, low noise"""
    rng = np.random.default_rng(seed)
    m = orc.Mode(mode, sample_rate=rate)
    out = []
    for _ in range(count):
        x, _ = lay_out(rng, m, transmission(rng, m, int(rng.integers(4, 8)), float(rng.uniform(0.3, 1.0))), 1e-3)
        out.append(x)
    return out


def fixed_per_candidate(monkeypatch, mode, rate, **kw):
    """an engine whose rx_batch runs the per-candidate kernel, as the tone calls do"""
    monkeypatch.setenv("FSK_B200_MULTI", "0")
    monkeypatch.setenv("FSK_B200_PREFIX", "0")
    e = mm().RxEngine.for_mode(mode, rate, **kw)
    monkeypatch.delenv("FSK_B200_MULTI")
    monkeypatch.delenv("FSK_B200_PREFIX")
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("key", KEYS, ids=[str(k) for k in KEYS])
def test_the_engine_pair_gives_the_fixed_tone_records(key, monkeypatch):
    """Every stream on the engine's own pair: records and states bit-identical to rx_batch on the
    per-candidate kernel (FSK_B200_MULTI=0 FSK_B200_PREFIX=0) of the same shape."""
    mode, rate = COVER[key]
    streams = preset_streams(mode, rate, 4, zlib.crc32(repr(key).encode()))
    fixed = fixed_per_candidate(monkeypatch, mode, rate)
    eng = mm().RxEngine.for_mode(mode, rate)
    p = eng.params
    bands = torch().tensor([[p.b_mark, p.b_space]] * len(streams), dtype=torch().int32).to(dev())
    assert bands.cpu().numpy().tolist()[0] == eng.tone_bands(float(p.f_mark), float(p.f_space), device=dev()).cpu().numpy()[0].tolist()
    buf, n = rows(streams, np.float32, 4)
    lens = np.array([a.size for a in streams], np.int32)
    fa, sa = run_tones(eng, buf, n, lens, bands)
    t = torch()
    fb, sb = fixed.rx_batch(upload(buf), nsamples=n, nsamples_each=upload(lens))
    sync()
    G, W, L = key
    assert fixed.last_kernel().startswith("k_rx<G=%d,W=%d,L=%d,mode=0(per-candidate)" % (G, W, L)), fixed.last_kernel()
    sa, sb = mm().states_to_numpy(sa), mm().states_to_numpy(sb)
    assert sa.tobytes() == sb.tobytes(), key
    fa, fb = mm().frames_to_numpy(fa), mm().frames_to_numpy(fb)
    for s in range(len(streams)):
        k = int(sa["nframes"][s])
        assert k >= 3 and fa[s, :k].tobytes() == fb[s, :k].tobytes(), (key, s)


@pytest.mark.gpu
def test_bell103_originate_and_answer_in_one_call():
    """Bell103 originate (1270/1070 Hz) and answer (2225/2025 Hz) streams in one call give the oracle's
    records on their pairs; a line carrying both directions summed, given once with each pair, gives both
    texts as the oracle decodes them."""
    streams, pairs, want = duplex_case()
    eng = mm().RxEngine.for_mode("300", 48000)
    bands = eng.tone_bands([p[0] for p in pairs], [p[1] for p in pairs], device=dev())
    buf, n = rows(streams, np.float32, 4)
    frames, states = run_tones(eng, buf, n, [a.size for a in streams], bands)
    assert "k_rx_tones<G=16,W=3,L=4," in eng.last_kernel()
    fr, st = mm().frames_to_numpy(frames), mm().states_to_numpy(states)
    out, cnt = eng.decode_batch(mm().DECODE_ASCII, frames, states)
    sync()
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    rx = orc.Mode("300", sample_rate=48000)
    for s, w in enumerate(want):
        recs = fr[s, :int(st["nframes"][s])]
        compare_frames(as_oracle_frames(recs), w["frames"], "duplex stream %d" % s)
        text = orc.decode_records(rx, "ascii8", orc.frame_records(w["frames"]))
        assert len(text) >= 5 and out[s, :cnt[s]].tobytes() == text, s
    assert out[6, :cnt[6]].tobytes() != out[7, :cnt[7]].tobytes()


# --------------------------------------------------------------------------
# edges
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_stream_without_a_valid_pair_is_skipped():
    """A band >= nbands: that stream gets no records and keeps its state byte for byte; its neighbours
    decode as they do without it."""
    t = torch()
    streams, pairs, _ = duplex_case()
    eng = mm().RxEngine.for_mode("300", 48000)
    nb = int(eng.params.nbands)
    good = eng.tone_bands([p[0] for p in pairs[:3]], [p[1] for p in pairs[:3]], device=dev())
    buf, n = rows(streams[:3], np.float32, 4)
    lens = [a.size for a in streams[:3]]
    fa, sa = run_tones(eng, buf, n, lens, good)
    for bad in ([nb, 5], [5, nb], [0xFFFFFFFF, 0xFFFFFFFF]):
        bands = good.clone()
        bands[1] = t.tensor(np.array(bad, np.uint32).view(np.int32)).to(bands.device)
        st0 = np.zeros(3, mm().STATE_DTYPE)
        st0["pos"][1], st0["carrier"][1], st0["track_amplitude"][1], st0["nframes"][1] = 1234, 1, 0.5, 2
        states = state_rows(st0)
        frames = t.full((3, eng.max_frames(n), 5), 0x5A5A5A5A, dtype=t.int32).to(dev())
        frames, sb = eng.rx_batch_tones(upload(buf), bands, nsamples=n, states=states,
                                        frames=frames, nsamples_each=upload(np.array(lens, np.int32)))
        sync()
        sb = mm().states_to_numpy(sb)
        assert sb[1].tobytes() == st0[1].tobytes(), bad
        assert (frames.cpu().numpy()[1] == 0x5A5A5A5A).all(), bad
        ra, rb = mm().frames_to_numpy(fa), mm().frames_to_numpy(frames)
        for s in (0, 2):
            k = int(mm().states_to_numpy(sa)["nframes"][s])
            assert sb[s].tobytes() == mm().states_to_numpy(sa)[s].tobytes() and ra[s, :k].tobytes() == rb[s, :k].tobytes()


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """-ENOTSUP for a mode the per-candidate kernel cannot take (0.5 baud) and -EINVAL for a NULL tone_bands,
    with no launch; an invalid pair raises on the host."""
    t = torch()
    L = mm().lib()
    x = t.zeros((2, 4096), dtype=t.float32).to(dev())
    fr = t.zeros((2, 16, 5), dtype=t.int32).to(dev())
    st = t.zeros((2, mm().STATE_WORDS), dtype=t.int32).to(dev())
    p = lambda a: C.c_void_p(a.data_ptr())
    slow = mm().RxEngine.for_mode("0.5", 48000)
    bands = slow.tone_bands([1000.0, 1400.0], [1200.0, 1600.0], device=dev())
    eng = mm().RxEngine.for_mode("1200", 48000)
    n0 = mm().launch_count()
    with pytest.raises(RuntimeError, match="-95"):
        slow.rx_batch_tones(x, bands, nsamples=4096)
    assert L.fsk_b200_rx_batch_tones(eng._e, p(x), 2, 4096, None, 4096, None, p(fr), 16, p(st), None) == -EINVAL
    assert L.fsk_b200_rx_batch_tones_s16(eng._e, p(x), 2, 4096, None, 4096, None, p(fr), 16, p(st), None) == -EINVAL
    assert L.fsk_b200_rx_batch_tones(eng._e, p(x), 2, 4096, None, 4097, p(bands), p(fr), 16, p(st), None) == -EINVAL
    assert mm().launch_count() == n0
    with pytest.raises(ValueError):
        eng.tone_bands([1200.0], [30000.0])
    with pytest.raises(ValueError):
        eng.tone_bands([-1200.0], [2200.0])


@pytest.mark.gpu
@pytest.mark.parametrize("src", ["f32", "s16"])
def test_output_overflow_resumes_to_the_records_of_one_pass(src):
    """Every call stops after 3 records and the next resumes from the saved state: the records of one pass."""
    t = torch()
    marks, spaces, streams, lens, _ = random_case("1200", 48000)
    eng = mm().RxEngine.for_mode("1200", 48000)
    bands = eng.tone_bands(marks, spaces, device=dev())
    buf, n = rows([pcm(a) for a in streams], np.int16, 8) if src == "s16" else rows(streams, np.float32, 4)
    fw, sw = run_tones(eng, buf, n, lens, bands)
    fw, sw = mm().frames_to_numpy(fw), mm().states_to_numpy(sw)
    whole = [[fw[s, i].tobytes() for i in range(int(sw["nframes"][s]))] for s in range(len(streams))]
    states = t.zeros((len(streams), mm().STATE_WORDS), dtype=t.int32).to(dev())
    got = [[] for _ in streams]
    for call in range(10000):
        frames, states = run_tones(eng, buf, n, lens, bands, states=states, max_frames=3)
        fr, st = mm().frames_to_numpy(frames), mm().states_to_numpy(states)
        for s in range(len(streams)):
            got[s] += [fr[s, i].tobytes() for i in range(int(st["nframes"][s]))]
        if (st["done"] == 1).all():
            break
        st["nframes"][:] = 0
        states = state_rows(st)
    assert call >= 2 and got == whole
    st["nframes"] = sw["nframes"]
    assert st.tobytes() == sw.tobytes()


@pytest.mark.gpu
def test_a_new_pair_takes_effect_at_the_call_position(monkeypatch):
    """A row carrying a Bell103 originate transmission and then an answer one: the first call on the
    originate pair stops where its samples end; the second call, on the answer pair, continues from that
    state exactly as a fixed-tone engine built for the answer pair does."""
    t = torch()
    rng = np.random.default_rng(7)
    mo, ma = on_pair("300", 48000, *ORIGINATE), on_pair("300", 48000, *ANSWER)
    a, b = transmission(rng, mo, 6, 0.7), transmission(rng, ma, 6, 0.7)
    x = np.concatenate([np.zeros(777, np.float32), a, np.zeros(3000, np.float32), b]).astype(np.float32)
    cut = 777 + a.size + 1500
    eng = mm().RxEngine.for_mode("300", 48000)
    bo = eng.tone_bands([ORIGINATE[0]] * 2, [ORIGINATE[1]] * 2, device=dev())
    ba = eng.tone_bands([ANSWER[0]] * 2, [ANSWER[1]] * 2, device=dev())
    buf, n = rows([x, x], np.float32, 4)
    f1, s1 = run_tones(eng, buf, n, [cut, cut], bo)
    s1 = mm().states_to_numpy(s1)
    assert (s1["done"] == 1).all() and int(s1["nframes"][0]) >= 6
    s1["done"][:] = 0
    s1["nframes"][:] = 0
    f2, s2 = run_tones(eng, buf, n, [x.size] * 2, ba, states=state_rows(s1))
    fixed = fixed_per_candidate(monkeypatch, "300", 48000, f_mark=ANSWER[0], f_space=ANSWER[1])
    f3, s3 = fixed.rx_batch(upload(buf), nsamples=n, states=state_rows(s1))
    sync()
    s2, s3 = mm().states_to_numpy(s2), mm().states_to_numpy(s3)
    assert s2.tobytes() == s3.tobytes()
    k = int(s2["nframes"][0])
    assert k >= 6 and mm().frames_to_numpy(f2)[:, :k].tobytes() == mm().frames_to_numpy(f3)[:, :k].tobytes()
    out, cnt = eng.decode_batch(mm().DECODE_ASCII, f2, state_rows(s2))
    want = orc.rx_run(ma, b, literal=False)["frames"]
    rx = orc.Mode("300", sample_rate=48000)
    assert out.cpu().numpy()[0, :int(cnt.cpu().numpy()[0])].tobytes() == orc.decode_records(
        rx, "ascii8", orc.frame_records(want))


# --------------------------------------------------------------------------
# live streams
# --------------------------------------------------------------------------
@pytest.mark.gpu
def test_live_receiver_with_tones_does_not_depend_on_the_cut():
    """LiveReceiver(tones=...) fed the duplex streams in random chunks prints, for every cut, the text of
    one rx_batch_tones call over the whole streams."""
    from minimodem_b200.serving import LiveReceiver
    t = torch()
    streams, pairs, _ = duplex_case()
    eng = mm().RxEngine.for_mode("300", 48000)
    bands = eng.tone_bands([p[0] for p in pairs], [p[1] for p in pairs], device=dev())
    buf, n = rows(streams, np.float32, 4)
    lens = np.array([a.size for a in streams], np.int64)
    frames, states = run_tones(eng, buf, n, lens, bands)
    out, cnt = eng.decode_batch(mm().DECODE_ASCII, frames, states)
    sync()
    whole = [out.cpu().numpy()[s, :int(cnt.cpu().numpy()[s])].tobytes() for s in range(len(streams))]
    assert all(len(w) >= 5 for w in whole)
    rng = np.random.default_rng(9)
    for max_chunk in (701, 5000):
        lr = LiveReceiver("300", 48000, len(streams), max_chunk=max_chunk, device=dev(), tones=bands)
        fed = np.zeros(len(streams), np.int64)
        texts = [b""] * len(streams)

        def take(res):
            o, c = res
            o, c = o.cpu().numpy(), c.cpu().numpy()
            return [texts[s] + o[s, :c[s]].tobytes() for s in range(len(streams))]
        while (fed < lens).any():
            k = np.minimum(rng.integers(1, max_chunk + 1, len(streams)), lens - fed)
            chunk = np.zeros((len(streams), max_chunk), np.float32)
            for s in range(len(streams)):
                chunk[s, :k[s]] = buf[s, fed[s]:fed[s] + k[s]]
            texts = take(lr.feed(upload(chunk), upload(k.astype(np.int32))))
            fed += k
        texts = take(lr.finish())
        assert texts == whole, max_chunk
