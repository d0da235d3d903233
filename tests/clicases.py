"""Helpers of the tests that run the reference CLI: random invocations, WAV files, and the emulation build
of the kernels under the product library's name (for the drop-in CLI on a machine without a GPU)."""
import os
import struct

import numpy as np

import orc

HERE = os.path.dirname(os.path.abspath(__file__))


def random_invocation(rng):
    """(mode, oracle Mode kwargs, --tx arguments, --rx arguments, float samples, volume) of a random reference
    CLI invocation: baud and sample rate, framing, bit order, inversion, tone pair and sample format"""
    while True:
        baud = int(rng.choice([75, 110, 150, 300, 600, 1200, 2400, 4800]))
        rate = int(rng.choice([8000, 11025, 16000, 22050, 44100, 48000]))
        if not (6 <= rate / baud <= 700):
            continue
        args, kw = [str(baud), "--samplerate", str(rate)], dict(sample_rate=rate)
        if rng.random() < 0.3:
            args = ["-7"] + args
            kw["n_data_bits"] = 7
        if rng.random() < 0.4:
            sb = int(rng.choice([1, 2, 3]))
            args += ["--startbits", str(sb)]
            kw["startbits"] = sb
        if rng.random() < 0.5:
            st = float(rng.choice([1.0, 1.5, 2.0]))
            args += ["--stopbits", str(st)]
            kw["stopbits"] = st
        for flag, key in (("--msb-first", "msb_first"), ("--invert-start-stop", "invert_start_stop"),
                          ("--inverted", "inverted")):
            if rng.random() < 0.25:
                args.append(flag)
                kw[key] = True
        if rng.random() < 0.3 and baud >= 400:
            mark = float(rng.choice([1000, 1300, 1500, 1800]))
            space = mark + float(rng.choice([400, 600, 1000]))
            if space < rate / 2 - 300:
                args += ["-M", str(mark), "-S", str(space)]
                kw["mark"], kw["space"] = mark, space
        flt = rng.random() < 0.3
        vol = float(rng.choice([1.0, 0.5, 0.1]))
        tx = args + (["--float-samples"] if flt else []) + (["--volume", str(vol)] if vol != 1.0 else [])
        try:
            m = orc.Mode(str(baud), **kw)
            m.derived()
            orc.Plan(m.sample_rate, m.mark_f, m.space_f, m.band_width)
        except Exception:
            continue
        if m.frame_n_bits > 12:            # longer frames hit the reference's ring limit (DESIGN.md 5, item 2)
            continue
        return str(baud), kw, tx, args, flt, vol


def write_wav(path, samples, rate, as_float):
    """a mono WAV the reference CLI reads: float32, or 16-bit PCM of samples * 32768"""
    if as_float:
        data, fmt, bits = samples.astype("<f4").tobytes(), 3, 32
    else:
        data, fmt, bits = np.round(samples * 32768.0).astype("<i2").tobytes(), 1, 16
    hdr = b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVE" + b"fmt " + struct.pack(
        "<IHHIIHH", 16, fmt, 1, rate, rate * bits // 8, bits // 8, bits) + b"data" + struct.pack("<I", len(data))
    with open(path, "wb") as f:
        f.write(hdr + data)


def emulation_as_product():
    """A directory in which the emulation build answers to the product library's name."""
    import emu_mode                             # tests/emu
    emu_mode.build()
    d = os.path.join(HERE, "emu", "as_product")
    os.makedirs(d, exist_ok=True)
    link = os.path.join(d, "libfsk_b200.so")
    if not os.path.islink(link):
        os.symlink(os.path.join("..", "libfsk_b200_emu.so"), link)
    return d
