"""The launch policy of the rx and find_frame calls, pinned.

For every configuration below -- a preset and sample rate, a call, the environment knobs that steer the
launcher and a stream count -- tests/launch_plans.json holds what the call picks: its last_kernel() string
(kernel instance, G, W, L, threads, ring, shared memory, blocks, look-ahead), whether an int16 call runs, or
the error it returns.  The rows are 16 zero samples long: the launch shape depends on the mode, the knobs
and the stream count, never on the samples.  A change of the launch policy fails here; regenerating the
fixture is then a deliberate, reviewable diff:

    FSK_B200_EMU=1 python tests/test_launch_plans.py --write

The host emulation (tests/emu) has the H100's opt-in shared memory, so its strings are the device's, except
that it always runs the prefix-table kernel's cp.async fill: a float-row prefix-table launch shows fill=1 on
the device (unless FSK_B200_PFX_FILL=0) where the fixture, written under the emulation, shows fill=0."""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "launch_plans.json")

PRESETS = ("1200", "300", "rtty", "tdd", "same", "callerid", "uic", "V.21", "0.5")
RATES = (8000, 48000)
CALLS = ("rx", "rx_s16", "s16_runs", "tones", "tones_k2", "auto", "find_frame")
SMEM_MAX = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (and of the emulation)
RING_OVER_SMEM = str(SMEM_MAX // 4 + 128)
PER_CAND = {"FSK_B200_MULTI": "0", "FSK_B200_PREFIX": "0"}
# the knob sets of the rx launch families (tests/rxfam.py), then one knob at a time
KNOB_SETS = [
    PER_CAND,
    dict(PER_CAND, FSK_B200_NO_SLIDE="1"),
    {"FSK_B200_MULTI": "2", "FSK_B200_PREFIX": "0"},
    {"FSK_B200_PREFIX": "1", "FSK_B200_PFX_FILL": "1"},
    {"FSK_B200_PREFIX": "1", "FSK_B200_PFX_FILL": "0"},
    {"FSK_B200_MULTI": "1"},
] + [{"FSK_B200_LANES": str(v)} for v in (4, 8, 16, 32)] \
  + [{"FSK_B200_SPLIT": str(v)} for v in (1, 2, 4)] \
  + [{"FSK_B200_WPB": str(v)} for v in (1, 2, 3, 4)] \
  + [{"FSK_B200_RING": v} for v in ("128", "16384", RING_OVER_SMEM)]
KNOBS = sorted({k for s in KNOB_SETS for k in s})
# the presets every knob set runs on: one per default kernel (per-candidate, prefix table) and SAME's 10 windows
KNOB_PRESETS = (("1200", 48000), ("300", 48000), ("rtty", 8000), ("same", 48000))
KNOB_CALLS = ("rx", "tones", "find_frame")
NSAMPLES = 16


def knob_key(env):
    return ",".join("%s=%s" % (k[len("FSK_B200_"):], v) for k, v in sorted(env.items())) or "default"


def configs(preset, rate):
    """(key, call, knob set, nstreams): every call under the default knobs for 7 streams, rx also for 1 and 257;
    on KNOB_PRESETS, KNOB_CALLS under every knob set"""
    cases = [(c, {}, 7) for c in CALLS] + [("rx", {}, 1), ("rx", {}, 257)]
    if (preset, rate) in KNOB_PRESETS:
        cases += [(c, env, 7) for env in KNOB_SETS for c in KNOB_CALLS]
    for c, env, n in cases:
        if c in ("rx", "rx_s16") and (preset == "0.5" or "FSK_B200_SPLIT" in env
                                      or env.get("FSK_B200_RING") == RING_OVER_SMEM):
            # where the rx calls may run the generic kernel: under the host emulation it stalls on rows
            # shorter than a search window (a million samples at 0.5 baud); the other calls pin these
            continue
        if c == "find_frame" and env.get("FSK_B200_LANES") == "4":
            # k_find_frame at G = 4 only with whole warps of streams: in a warp that holds fewer than
            # 8 streams its search waits in a warp-wide sync the missing streams never reach
            n = (n + 7) & ~7
        yield "%s@%d %s/%s/n=%d" % (preset, rate, c, knob_key(env), n), c, env, n


def as_emulated(s, env):
    """a device launch string as the host emulation shows it (its prefix-table float rows take the cp.async fill)"""
    if env.get("FSK_B200_PFX_FILL") != "0":
        s = s.replace("mode=3(prefix-table),fill=1,src=f32", "mode=3(prefix-table),fill=0,src=f32")
    return s


def plan(mm, torch, dev, preset, rate, call, env, n):
    """what `call` on n streams of an engine for (preset, rate) made under `env` launches, as one string"""
    saved = {k: os.environ.pop(k, None) for k in KNOBS}
    os.environ.update(env)
    try:
        eng = mm.RxEngine.for_mode(preset, rate)            # the knobs are read here
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v
    try:
        if call == "s16_runs":
            return "s16_runs=%s" % eng.rx_batch_s16_runs(n)
        dt = torch.int16 if call == "rx_s16" else torch.float32
        x = torch.zeros((n, NSAMPLES), dtype=dt, device=dev)
        if call in ("rx", "rx_s16"):
            eng.rx_batch(x)
        elif call.startswith("tones"):
            k = 2 if call == "tones_k2" else 1
            cfg = mm.rx_config_for_mode(preset, rate)
            bands = eng.tone_bands([cfg.f_mark] * (n * k), [cfg.f_space] * (n * k), device=dev)
            eng.rx_batch_tones(x, bands, channels_per_row=k)
        elif call == "auto":
            eng.set_auto_carrier()
            eng.rx_batch_auto(x)
        else:
            i32 = lambda v: torch.full((n,), v, dtype=torch.int32, device=dev)
            eng.find_frame_batch(x, i32(0), i32(0), i32(1), i32(1),
                                 torch.full((n,), 2.3, device=dev))
        return as_emulated(eng.last_kernel(), env)
    except RuntimeError as e:
        return "error: %s" % e
    finally:
        eng.destroy()


def plans(preset, rate):
    import minimodem_b200 as mm
    import torch
    import gpudev
    out = {key: plan(mm, torch, gpudev.dev(), preset, rate, c, env, n) for key, c, env, n in configs(preset, rate)}
    gpudev.sync()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("preset", PRESETS)
def test_launch_plan(preset, rate):
    pytest.importorskip("torch")
    with open(FIXTURE) as f:
        want = {k: v for k, v in json.load(f).items() if k.startswith("%s@%d " % (preset, rate))}
    got = plans(preset, rate)
    assert sorted(got) == sorted(want)
    bad = ["%s:\n  got  %s\n  want %s" % (k, got[k], want[k]) for k in sorted(got) if got[k] != want[k]]
    assert not bad, "%d of %d launches differ:\n%s" % (len(bad), len(got), "\n".join(bad[:20]))


def write():
    """tests/launch_plans.json from the library as built (run under FSK_B200_EMU=1)"""
    sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.join(HERE, "emu")]
    import conftest  # noqa: F401  (selects the emulation under FSK_B200_EMU=1)
    out = {}
    for p in PRESETS:
        for r in RATES:
            out.update(plans(p, r))
    with open(FIXTURE, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("%s: %d launches" % (FIXTURE, len(out)))


if __name__ == "__main__" and sys.argv[1:] == ["--write"]:
    write()
