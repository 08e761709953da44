"""CPU tier of the drop-in boundary: the relinked chain runtime loads, CPU effects still work through
it, and a GPU effect fails its init() loudly (returns NULL -> chain build fails) without a device."""
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DROPIN = os.path.join(ROOT, "oracle", "_ref", "dropin", "libdsp_dropin.so")
SHIM = os.path.join(ROOT, "oracle", "_ref", "shim")


def test_dropin_library_without_gpu():
    if not os.path.exists(DROPIN):
        pytest.skip("drop-in harness not built (needs the reference sources at build time)")
    import dsp_b200
    from oracle import ref
    c = ref.RefChain("remix 1 0", 48000, 2, lib_path=DROPIN)      # reference remix.c, still CPU: swaps the channels
    x = np.stack([np.ones(16), np.zeros(16)], axis=1)
    y = c.run(x)
    assert np.array_equal(y[:, 0], x[:, 1]) and np.array_equal(y[:, 1], x[:, 0])
    c.close()
    if dsp_b200.device_count() < 1:
        with pytest.raises(ValueError):
            ref.RefChain("eq 1k 1.0 3", 48000, 2, lib_path=DROPIN)
        # "!" lets an effect fail without aborting the chain build (effects_chain.c:455-458)
        c = ref.RefChain("remix 1 0 ! eq 1k 1.0 3", 48000, 2, lib_path=DROPIN)
        assert c.effect_names() == ["remix"]


def test_shim_exports_reference_symbols():
    """The replacement objects export exactly the symbols the reference's biquad.o fir.o fir_p.o hilbert.o
    resample.o export (SURVEY.md 8b)."""
    import subprocess
    objdir = os.path.join(SHIM, "obj")
    if not os.path.isdir(objdir):
        pytest.skip("shim objects not built")
    want = {"biquad.o": {"biquad_effect_init", "biquad_init", "biquad_reset", "biquad_init_using_type"},
            "gain.o": {"gain_effect_init"},
            "fir.o": {"fir_effect_init", "fir_effect_init_with_filter"},
            "fir_p.o": {"fir_p_effect_init", "fir_p_effect_init_with_filter"},
            "hilbert.o": {"hilbert_effect_init"}, "resample.o": {"resample_effect_init"}}
    for obj, syms in want.items():
        out = subprocess.run(["nm", "-g", "--defined-only", os.path.join(objdir, obj)], stdout=subprocess.PIPE, text=True).stdout
        have = {line.split()[-1] for line in out.splitlines() if " T " in line}
        assert syms <= have, (obj, syms - have)


def test_align_entry_point_and_fallback_symbols():
    """shim/align.c takes over align_effect_insert (align.h:27); the reference's align.o stays linked under
    ref_align_effect_insert (renamed with objcopy) as the host implementation for chains without GPU effects."""
    import subprocess
    obj, ref = os.path.join(SHIM, "obj", "align.o"), os.path.join(SHIM, "ref", "align.o")
    if not (os.path.exists(obj) and os.path.exists(ref)):
        pytest.skip("shim objects not built")
    nm = lambda p: {l.split()[-1] for l in subprocess.run(["nm", "-g", "--defined-only", p], stdout=subprocess.PIPE, text=True).stdout.splitlines() if " T " in l}
    assert "align_effect_insert" in nm(obj)
    assert nm(ref) == {"ref_align_effect_insert"}


def test_cpu_chains_keep_the_reference_align(have_ref):
    """A chain without GPU effects that needs alignment (delay.c hands its whole-sample part to the align pass,
    delay.c:153-157,199) gets the reference's own align effect through the fallback -- same output as the pure
    reference, no device needed."""
    if not os.path.exists(DROPIN) or not have_ref:
        pytest.skip("drop-in harness / compiled reference not built")
    from oracle import ref
    chain = ":0 delay 37S : remix 0 1"
    x = np.random.default_rng(0).standard_normal((500, 2))
    a = ref.RefChain(chain, 48000, 2)
    b = ref.RefChain(chain, 48000, 2, lib_path=DROPIN)
    assert a.effect_names() == b.effect_names()
    ya, ca = a.process(x, 128)
    yb, cb = b.process(x, 128)
    assert ca == cb and np.array_equal(ya, yb)


def test_frontend_library_and_ladspa_plugin_load():
    """The drop-in as a library (shim/frontend.c) and as the reference's LADSPA plugin (ladspa_dsp.c unmodified):
    both load and expose their entry points; without a device a GPU effect makes the chain build fail (no fallback)."""
    import dsp_b200
    from dsp_b200 import frontend
    if not frontend.available():
        pytest.skip("frontend library not built (needs the reference sources at build time)")
    L = frontend.lib()
    for n in ("dspfront_chain_new", "dspfront_chain_run", "dspfront_chain_time", "dspfront_chain_free"):
        assert hasattr(L, n)
    c = frontend.DropinChain("remix 1 0", 48000, 2)       # reference effect through the library frontend
    y = c.run(np.stack([np.ones(8), np.zeros(8)], axis=1))
    assert np.array_equal(y[:, 1], np.ones(8))
    c.close()
    if dsp_b200.device_count() < 1:
        with pytest.raises(ValueError):
            frontend.DropinChain("eq 1k 1.0 3", 48000, 2)
    plugin = os.path.join(ROOT, "oracle", "_ref", "dropin", "ladspa_dsp_b200.so")
    if os.path.exists(plugin):
        # in a child process: the plugin reads its configuration once, when it is loaded, and stays loaded for the rest
        # of the process -- tests/test_gpu_dropin.py loads it again with a configuration of its own
        import subprocess
        import sys
        env = dict(os.environ)
        env.setdefault("LADSPA_DSP_CONFIG_PATH", "/nonexistent")
        code = "import ctypes, sys; sys.exit(0 if hasattr(ctypes.CDLL(sys.argv[1]), 'ladspa_descriptor') else 1)"
        assert subprocess.run([sys.executable, "-c", code, plugin], env=env).returncode == 0


def test_mirror_reads_numbers_as_strtod():
    """dsp_b200.effects reads numeric words as the reference's strtod() + CHECK_ENDPTR do: decimal and hexadecimal
    forms, inf and nan, and nothing after the number (Python's float() also takes digit separators, strtod() does not)."""
    from dsp_b200.effects import ChainSyntaxError, parse_freq, parse_num, parse_width
    for word, want in (("3", 3.0), ("-3.5", -3.5), ("+.5", 0.5), ("1.", 1.0), ("1e3", 1000.0), ("2.5E-1", 0.25),
                       ("0x1.8p-1", 0.75), ("-0X10", -16.0), ("0x.8", 0.5), ("inf", float("inf")), ("-Infinity", float("-inf"))):
        assert parse_num(word) == want, word
    assert np.isnan(parse_num("nan")) and np.isnan(parse_num("NaN(1)"))
    for word in ("1_000", "", "x", "1e", "0x", "1 ", "3dB", "0x1p", "infin", "1.2.3"):
        with pytest.raises(ChainSyntaxError):
            parse_num(word)
    assert parse_freq("0x1p10k") == 1024000.0 and parse_width("0x1p1q") == (2.0, 1)
    for word in ("1_0k", "1kk"):
        with pytest.raises(ChainSyntaxError):
            parse_freq(word)
