"""GPU tier: every option form of the drop-in effects (shim/biquad.c, hilbert.c, resample.c, gain.c and the FIR
effects), run through the reference's own chain runtime against the pure reference (oracle/_ref/libdspref.so), the
biquad designs also against a long-double truth, and the Python mirror (dsp_b200.effects) against the drop-in.

The shim re-implements the reference's argument handling (biquad.c:27-89 and 441-533, hilbert.c:28-92,
resample.c:213-259, gain.c:80-141), and so does the mirror: a form one of them read differently would change the
audio.  Each case below drives one chain string through both libraries on 4 channels of about 3 x 8192 frames
(the four bq_inputs signals; for designs near Nyquist the first channel is a +-0.5 Nyquist tone instead), three
times: in 1024-frame calls (K1's split form), in 4096-frame calls (its 16-warp form), and in ragged calls after
a reset() that follows 5000 frames.  Then it drains.  Each pass must show the reference's effect list (or the one
device effect the shim merges a run into), its per-call frame counts with the drain, unselected channels equal
to the input bit for bit, and:
  - biquad designs: per selected channel accuracy.biquad_within_ref against the long-double cascade of the
    coefficients the table gives as numbers (ref.biquad_design(...) or b/a0), and the pure reference's own output
    within 1e-7 of that truth, relative to rms(truth) -- that shows the table reads the arguments as the
    reference does;
  - biquad -r: per channel nerr(gpu, ref) <= 1e-13;
  - gain / mult / add alone: bit-identical; merged runs within 1e-15;
  - hilbert, fir, fir_p, resample: nerr(gpu, ref) <= 1e-13.
Every refused form must make both libraries refuse the chain (ValueError), and the mirror too.  The absorb test
checks that a device chain absorbing another after it has run keeps both cascades' state.

Measured on an H100 80GB HBM3 (700 W limit), worst over the cases: biquad designs err_gpu at most 0.91 of its bound
(a 40 kHz bandpass at 192 kHz, where the bound is 64 u rms(truth)); largest err_gpu 4.7e-11 relative, on 1 Hz at
44.1 kHz; the pure reference's own error at most 6.2e-9.  The sections near Nyquist land at the FP64 recurrence's
error: highpass 47 kHz, Q 39 at 96 kHz 4.4e-13 against 4.3e-13 (before K1 summed each chunk's dot product in order
it was 2.2e-12).  biquad -r 4.0e-14; gain, mult and add bit-identical, merged runs 1.1e-16; hilbert 9.7e-16; fir
and fir_p 6.7e-16; resample 9.5e-15.  The Python mirror equals the drop-in bit for bit on every form it supports
except the biquads, which it fuses into one cascade (the same bounds hold).

Errors of each case are appended as JSON lines to the file DSP_B200_ACCURACY_LOG names, when it is set.
"""
import os

import numpy as np
import pytest

from accuracy import biquad_truth, biquad_within_ref, nerr
from test_gpu_accuracy import _record, bq_inputs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "oracle", "_ref", "dropin", "libdsp_dropin.so")
REFLIB = os.path.join(ROOT, "oracle", "_ref", "libdspref.so")
C = 4
N = 3 * 8192 + 5
RAGGED = [1, 2047, 2049, 4096, 5000, 1, 3000, 8191]      # then the rest of the stream
REF_TRUTH = 1e-7      # the pure reference's FP64 recurrence against the long-double truth, relative to rms(truth)
TOL = 1e-13
MERGED_TOL = 1e-15

Q, SLOPE, SLOPE_DB, OCT, HZ = 1, 2, 3, 4, 5
# width word -> (width, width type) as biquad.c:27-89 reads it; bw<order>[.<index>] as its pole pair's Q
WIDTHS = [("0.7", 0.7, Q), ("2.5q", 2.5, Q), ("1.5o", 1.5, OCT), ("250h", 250.0, HZ), ("1.2k", 1200.0, HZ),
          ("bw2", 0.7071067811865476, Q), ("bw4.0", 0.541196100146197, Q), ("bw4.1", 1.3065629648763766, Q),
          ("bw5.1", 1.618033988749895, Q), ("bw8.3", 2.5629154477415064, Q)]
SHELF_WIDTHS = [("0.8s", 0.8, SLOPE), ("12d", 12.0, SLOPE_DB)]
# (rate, f0 word, f0, near Nyquist): 1 Hz up to just below fs/2, plain and with k
FREQS = [(44100, "1", 1.0, False), (48000, "2.5k", 2500.0, False), (96000, "47k", 47000.0, True),
         (192000, "95k", 95000.0, True), (44100, "22000", 22000.0, True), (48000, "100", 100.0, False),
         (192000, "10", 10.0, False), (96000, "12.5k", 12500.0, False), (44100, "21.5k", 21500.0, True),
         (48000, "23.9k", 23900.0, True), (192000, "40k", 40000.0, False), (44100, "5k", 5000.0, False)]
BQ_TYPES = {"lowpass_1": 1, "highpass_1": 2, "allpass_1": 3, "lowshelf_1": 4, "highshelf_1": 5, "lowpass_1p": 6,
            "lowpass": 7, "highpass": 8, "bandpass_skirt": 9, "bandpass_peak": 10, "notch": 11, "allpass": 12, "eq": 13,
            "lowshelf": 14, "highshelf": 15, "lowpass_transform": 16, "highpass_transform": 17, "linkwitz_transform": 17}

CASES = {}


def _case(name, chain, fs, kind, tol=None, sections=None, touched=None, hf=False, fx=None, mirror=True):
    """kind: "bq" (value check against the long-double truth of `sections`), "riir", "exact" or "near" (against the
    pure reference within `tol`).  sections: [(coefficient spec, channels or None)] in chain order, a spec being
    ("d", type, arg0, arg1, arg2, arg3, width type) for ref.biquad_design at the case's rate or ("c", c0..c4).
    touched: the channels the chain may change (None: all; for "bq" the union of the sections').  fx: the drop-in's
    effect list where the shim merges a run into one device effect (None: the reference's).  mirror: whether
    dsp_b200.effects builds the chain (else it must raise ChainSyntaxError or NotImplementedError)."""
    assert name not in CASES, name
    if kind == "bq":
        chans = set()
        for _, ch in sections:
            chans |= set(range(C) if ch is None else ch)
        touched = sorted(chans)
    CASES[name] = dict(chain=chain, fs=fs, kind=kind, tol=tol, sections=sections, touched=list(range(C)) if touched is None else touched,
                       hf=hf, fx=fx, mirror=mirror)


def _d(t, a0, a1=0.0, a2=0.0, a3=0.0, wt=Q):
    return ("d", t, a0, a1, a2, a3, wt)


# -- 1. the biquad family, every width form each name accepts ---------------------------------------------------
_k = 0
for _name in ("lowpass_1", "highpass_1", "allpass_1", "lowshelf_1", "highshelf_1", "lowpass_1p"):
    for _fs, _fw, _f, _hf in (FREQS[_k % len(FREQS)], FREQS[(_k + 5) % len(FREQS)]):
        _g = 15.0 if _k % 2 else -15.0
        _args = "%s %g" % (_fw, _g) if _name.endswith("shelf_1") else _fw
        _a2 = _g if _name.endswith("shelf_1") else 0.0
        _case("%s/%s@%d" % (_name, _args.replace(" ", "_"), _fs), "%s %s" % (_name, _args), _fs, "bq",
              sections=[(_d(BQ_TYPES[_name], _f, 0.0, _a2), None)], hf=_hf)
        _k += 1
for _name in ("lowpass", "highpass", "bandpass_skirt", "bandpass_peak", "notch", "allpass", "eq", "lowshelf", "highshelf"):
    for _ww, _w, _wt in WIDTHS + (SHELF_WIDTHS if _name.endswith("shelf") else []):
        _fs, _fw, _f, _hf = FREQS[_k % len(FREQS)]
        if _wt == OCT and _hf:
            _fs, _fw, _f, _hf = FREQS[(_k + 1) % len(FREQS)]     # an octave width near Nyquist puts both poles at +-1
        if _name == "lowshelf" and _wt == SLOPE_DB and _f > _fs / 8:
            _fs, _fw, _f, _hf = (48000, "300", 300.0, False)     # slope in dB moves a low shelf's f0 up by 10^(|gain| / 80 / s)
        _k += 1
        _g = 15.0 if _k % 2 else -15.0
        _has_gain = _name in ("eq", "lowshelf", "highshelf")
        _args = "%s %s %g" % (_fw, _ww, _g) if _has_gain else "%s %s" % (_fw, _ww)
        _case("%s/%s@%d" % (_name, _args.replace(" ", "_"), _fs), "%s %s" % (_name, _args), _fs, "bq",
              sections=[(_d(BQ_TYPES[_name], _f, _w, _g if _has_gain else 0.0, 0.0, _wt), None)], hf=_hf)
for _name in ("lowpass_transform", "highpass_transform", "linkwitz_transform"):
    for _fs, _args, _v in ((48000, "30 0.707 10 0.5", (30.0, 0.707, 10.0, 0.5)),
                           (44100, "1k 2q 200 bw2", (1000.0, 2.0, 200.0, 0.7071067811865476)),
                           (192000, "20 bw4.1 40 0.5q", (20.0, 1.3065629648763766, 40.0, 0.5)),
                           (96000, "5k bw8.3 2.5k 0.7", (5000.0, 2.5629154477415064, 2500.0, 0.7))):
        _case("%s/%s@%d" % (_name, _args.replace(" ", "_"), _fs), "%s %s" % (_name, _args), _fs, "bq",
              sections=[(_d(BQ_TYPES[_name], *_v), None)])
# deemph: the high shelf presets of biquad.c:497-515
_case("deemph@44100", "deemph", 44100, "bq", sections=[(_d(15, 5283.0, 0.4845, -9.477, 0.0, SLOPE), None)])
_case("deemph@48000", "deemph", 48000, "bq", sections=[(_d(15, 5356.0, 0.479, -9.62, 0.0, SLOPE), None)])
# raw biquad b0 b1 b2 a0 a1 a2 -> b / a0 (a0 = 2 halves exactly); both poles at 0
_case("biquad/a0=2", "biquad 0.2 0.3 0.1 2 -1.2 0.5", 48000, "bq", sections=[(("c", 0.1, 0.15, 0.05, -0.6, 0.25), None)])
_case("biquad/poles_at_0", "biquad 0.5 -0.25 0.125 1 0 0", 96000, "bq", sections=[(("c", 0.5, -0.25, 0.125, 0.0, 0.0), None)])
# selectors, and runs the shim merges into one device effect
_case("sel/eq:0,2", ":0,2 eq 1k 1.0 15", 48000, "bq", sections=[(_d(13, 1000.0, 1.0, 15.0), (0, 2))])
_case("sel/highshelf:1-", ":1- highshelf 8k 0.8s -15", 44100, "bq", sections=[(_d(15, 8000.0, 0.8, -15.0, 0.0, SLOPE), (1, 2, 3))])
_case("sel/two_selectors", ":0,2 eq 1k 1.0 15 :1- highpass 40 bw4.1 :", 96000, "bq",
      sections=[(_d(13, 1000.0, 1.0, 15.0), (0, 2)), (_d(8, 40.0, 1.3065629648763766), (1, 2, 3))], fx=["eq"])
_case("merge/four_sections", "eq 1k 1.0 3 lowshelf 200 0.7 -2 highpass 30 bw4.0 highpass 30 bw4.1", 48000, "bq",
      sections=[(_d(13, 1000.0, 1.0, 3.0), None), (_d(14, 200.0, 0.7, -2.0), None), (_d(8, 30.0, 0.541196100146197), None),
                (_d(8, 30.0, 1.3065629648763766), None)], fx=["eq"])
_case("merge/selected_run", ":3 lowpass_1 2k notch 10k 3q :0-2 highshelf_1 15k 6", 192000, "bq",
      sections=[(_d(1, 2000.0), (3,)), (_d(11, 10000.0, 3.0), (3,)), (_d(5, 15000.0, 0.0, 6.0), (0, 1, 2))], fx=["lowpass_1"])
_case("merge/gain_and_eq", "gain -6 eq 100 0.7 15 eq 5k 2q -15", 44100, "bq",
      sections=[(("c", 10 ** (-6 / 20.0), 0.0, 0.0, 0.0, 0.0), None), (_d(13, 100.0, 0.7, 15.0), None), (_d(13, 5000.0, 2.0, -15.0), None)],
      fx=["gain"])

# -- 2. biquad -r: the reference's reverse-IIR design, run as a device FIR ---------------------------------------
for _name, _args in (("lowpass_1", "2k"), ("highpass_1", "1k"), ("allpass_1", "3k"), ("lowshelf_1", "1k 6"), ("highshelf_1", "2k -6"),
                     ("lowpass_1p", "5k"), ("lowpass", "2k 0.7"), ("highpass", "1k bw2"), ("bandpass_skirt", "3k 1o"),
                     ("bandpass_peak", "2k 500h"), ("notch", "4k 1q"), ("allpass", "1.5k 0.6"), ("eq", "2k 1.0 6"),
                     ("lowshelf", "1k 0.8s 4"), ("highshelf", "3k 6d -4"), ("lowpass_transform", "2k 0.7 1k 0.5"),
                     ("highpass_transform", "1k 0.7 2k 0.5"), ("linkwitz_transform", "1k 0.5 2k 0.7"), ("deemph", ""),
                     ("biquad", "0.2 0.3 0.1 2 -1.2 0.5")):
    _case("riir/%s" % _name, ("%s -r %s" % (_name, _args)).strip(), 48000, "riir", mirror=False)
for _t in (10, 80, 200):
    _case("riir/eq_-r%d" % _t, "eq -r%d 2k 1.0 6" % _t, 48000, "riir", mirror=False)
_case("riir/two_channels", ":0 highpass -r 2k bw2 :2 lowpass -r 3k 0.7 :", 48000, "riir", touched=[0, 2], mirror=False)

# -- 3. gain / mult / add -----------------------------------------------------------------------------------------
for _name, _chain, _touched in (("gain", "gain -3", None), ("gain:0,2", ":0,2 gain 6", [0, 2]), ("mult:1-", ":1- mult 0.3", [1, 2, 3]),
                                ("mult", "mult -2", None), ("add:0,2", ":0,2 add 0.25", [0, 2]), ("add:3", ":3 add -0.125", [3]),
                                ("add", "add 1e-3", None), ("mult_hex", "mult 0x1.8p-1", None)):
    _case("gain/" + _name, _chain, 48000, "exact", touched=_touched)
_case("gain/merged_gain", "gain 3 gain -3", 48000, "near", tol=MERGED_TOL)
_case("gain/merged_mult", "mult 2 :1 mult 0.5 :", 48000, "near", tol=MERGED_TOL)
_case("gain/merged_add_gain", "add 0.25 gain -6", 48000, "near", tol=MERGED_TOL, fx=["add"])

# -- 4. hilbert: 15 taps is fir's direct form (latency 0), 17 its FFT form (latency len) ---------------------------
for _chain in ("hilbert 5", "hilbert 15", "hilbert 17", "hilbert 255", "hilbert 1025", "hilbert -a 0 255", "hilbert -a 45 17",
               "hilbert -a -90 15", "hilbert -a 90 255", "hilbert -a 180 1025", "hilbert -a 30.5 255", "hilbert -p 255",
               "hilbert -p -a 45 1025", "hilbert -z 255", ":1,3 hilbert -a 30.5 17"):
    _case(_chain.replace(" ", "_"), _chain, 48000, "near", tol=TOL, touched=[1, 3] if _chain.startswith(":1,3") else None)
for _chain in ("hilbert -c 255", "hilbert -p -c 17"):
    _case(_chain.replace(" ", "_"), _chain, 48000, "near", tol=TOL, mirror=False)

# -- 5. fir / fir_p from coefs: (<= 16 taps: fir's direct form, fir.c:239) ------------------------------------------
_rng = np.random.default_rng(77)
FIR_TAPS = {n: _rng.uniform(-1, 1, n) * np.exp(-np.arange(n) / (0.3 * n + 1)) for n in (1, 16, 17, 300)}
for _eff in ("fir", "fir_p"):
    for _n, _h in FIR_TAPS.items():
        _case("%s/coefs%d" % (_eff, _n), "%s coefs:%s" % (_eff, ",".join("%.17g" % v for v in _h)), 48000, "near", tol=TOL)
    _h2 = _rng.uniform(-1, 1, (40, 2))
    _case("%s/two_columns:1,2" % _eff, ":1,2 %s coefs:%s/%s" % (_eff, ",".join("%.17g" % v for v in _h2[:, 0]), ",".join("%.17g" % v for v in _h2[:, 1])),
          48000, "near", tol=TOL, touched=[1, 2])

# -- 6. resample -----------------------------------------------------------------------------------------------------
for _fs, _args in ((44100, "48k"), (44100, "48000"), (48000, "44.1k"), (44100, "0.7 48k"), (48000, "0.999 96000"), (48000, "x2"),
                   (44100, "x3"), (96000, "/2"), (48000, "/3"), (48000, "48000")):
    _case("resample/%s@%d" % (_args.replace(" ", "_"), _fs), "resample " + _args, _fs, "near", tol=TOL)

# -- 7. refusals: (chain, rate, the reference check that refuses it, whether to run the pure reference) ------------
REFUSALS = {
    "f0_at_nyquist": ("lowpass 22050 0.7", 44100, "biquad.c:474 GET_FREQ_ARG -> CHECK_FREQ (util.h:36-37: f0 < fs/2)", True),
    "f0_at_nyquist_k": ("lowpass_1 24k", 48000, "biquad.c:458 CHECK_FREQ", True),
    "fp_at_nyquist": ("lowpass_transform 30 0.7 48k 0.5", 96000, "biquad.c:493 CHECK_FREQ on fp", True),
    "width_0": ("eq 1k 0 3", 48000, "biquad.c:422 CHECK_RANGE(width > 0)", True),
    "slope_on_eq": ("eq 1k 0.5s 3", 48000, "biquad.c:484 CHECK_WIDTH_TYPE(no slope) on eq", True),
    "slope_db_on_lowpass": ("lowpass 1k 12d", 48000, "biquad.c:476 CHECK_WIDTH_TYPE(no slope)", True),
    "oct_on_transform": ("lowpass_transform 30 1o 10 0.5", 48000, "biquad.c:492 CHECK_WIDTH_TYPE(Q) on width_z", True),
    "hz_on_transform": ("highpass_transform 30 0.7 10 20h", 48000, "biquad.c:495 CHECK_WIDTH_TYPE(Q) on width_p", True),
    "bw1": ("lowpass 1k bw1", 48000, "biquad.c:36-38 parse_width: order < 2", True),
    "bw4.2": ("lowpass 1k bw4.2", 48000, "biquad.c:47-50 parse_width: index out of range", True),
    "bw5.2": ("highpass 1k bw5.2", 48000, "biquad.c:47-50 parse_width: index >= order / 2", True),
    "bw4.": ("lowpass 1k bw4.", 48000, "biquad.c:45-46 parse_width: no index after the dot", True),
    "width_trailing": ("lowpass 1k 0.7qx", 48000, "biquad.c:421 CHECK_ENDPTR after the width suffix", True),
    "f0_trailing": ("eq 1kz 0.7 3", 48000, "biquad.c:414 CHECK_ENDPTR after parse_freq's k", True),
    "gain_trailing": ("eq 1k 0.7 3dB", 48000, "biquad.c:408 GET_ARG CHECK_ENDPTR on gain", True),
    "thresh_9": ("eq -r9 1k 0.7 3", 48000, "biquad.c:394 CHECK_RANGE(10 <= thresh <= 200)", True),
    "thresh_201": ("eq -r201 1k 0.7 3", 48000, "biquad.c:394 CHECK_RANGE(10 <= thresh <= 200)", True),
    "thresh_x": ("eq -rx 1k 0.7 3", 48000, "biquad.c:393 CHECK_ENDPTR on thresh", True),
    "eq_two_args": ("eq 1k 0.7", 48000, "biquad.c:434 INIT_COMMON: argc - ind != 3", True),
    "lowpass_three_args": ("lowpass 1k 0.7 3", 48000, "biquad.c:434 INIT_COMMON: argc - ind != 2", True),
    "biquad_five_args": ("biquad 1 0 0 1 0", 48000, "biquad.c:434 INIT_COMMON: argc - ind != 6", True),
    "deemph_arg": ("deemph 1", 48000, "biquad.c:434 INIT_COMMON: argc - ind != 0", True),
    "deemph_96k": ("deemph", 96000, "biquad.c:511-513 sample rate must be 44100 or 48000", True),
    "hilbert_3": ("hilbert 3", 48000, "hilbert.c:57-60 taps must be > 3", True),
    "hilbert_256": ("hilbert 256", 48000, "hilbert.c:61-64 taps must be odd", True),
    "hilbert_angle_x": ("hilbert -a x 255", 48000, "hilbert.c:43 CHECK_ENDPTR on angle", True),
    "hilbert_no_taps": ("hilbert -p", 48000, "hilbert.c:50 g.ind != argc - 1", True),
    "gain_trailing_db": ("gain 3dB", 48000, "gain.c:97 CHECK_ENDPTR on gain", True),
    "mult_two_args": ("mult 2 3", 48000, "gain.c:88 argc != 2", True),
    "gain_digit_separator": ("gain 1_0", 48000, "gain.c:97 CHECK_ENDPTR: strtod stops at the underscore", True),
    "resample_bw_0.5": ("resample 0.5 48k", 44100, "resample.c:233 CHECK_RANGE(0.7 <= bandwidth <= 0.999)", True),
    "resample_div_11": ("resample /11", 44100, "resample.c:242-245 11 is not a factor of 44100", True),
    # the pure reference divides by zero here (resample.c:242: fs % rate_div); only the drop-in is asked
    "resample_div_0": ("resample /0", 44100, "resample.c:242 rate_div = 0 (the shim refuses it before the modulo)", False),
    "resample_rate_0": ("resample 0", 44100, "resample.c:252 CHECK_RANGE(rate > 0)", True),
}


@pytest.fixture(scope="module")
def libs(gpu_lib):
    for p in (DROPIN, REFLIB):
        if not os.path.exists(p):
            pytest.fail("%s missing (built by __graft_entry__.build() where the reference sources exist)" % p)
    from oracle import ref
    return ref


def _input(case):
    x = bq_inputs(case["fs"], N, seed=len(case["chain"]))
    if case["hf"]:
        x[:, 0] = 0.5 * (1 - 2 * (np.arange(N) % 2))     # +-0.5 at fs/2
    return x


def _coefs(ref, case):
    """[S, C, 5] from the table: identity sections on the channels a section does not select."""
    secs = case["sections"]
    out = np.zeros((len(secs), C, 5))
    out[:, :, 0] = 1.0
    for s, (spec, ch) in enumerate(secs):
        c5 = ref.biquad_design(spec[1], case["fs"], *spec[2:]) if spec[0] == "d" else np.array(spec[1:], dtype=np.float64)
        for c in (range(C) if ch is None else ch):
            out[s, c] = c5
    return out


def _ragged_cuts():
    cuts = [0]
    for f in RAGGED:
        cuts.append(min(cuts[-1] + f, N))
    return cuts + [N] if cuts[-1] < N else cuts


def _pass(rc, x, how):
    """(output, per-call frame counts with the drain) of one pass through RefChain `rc`."""
    if how == "ragged":
        for i in range(0, 5000, 1024):
            rc.run(x[i:min(i + 1024, 5000)])
        rc.reset()
        cuts, block = _ragged_cuts(), 4096
    else:
        block = 1024 if how == "1024" else 4096
        cuts = list(range(0, N, block)) + [N]
    outs = [rc.run(x[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    outs += rc.drain(block)
    return np.concatenate(outs, axis=0), [y.shape[0] for y in outs]


def _check_values(name, case, how, y, want, x, truth=None, coefs=None):
    """The value checks of the case's kind; `want` is the pure reference's stream of the same pass."""
    kind, sel = case["kind"], case["touched"]
    if kind == "bq":
        rows = biquad_within_ref(y[:, sel], x[:, sel], coefs[:, sel], truth=truth[:, sel], ref64=want[:, sel])
        for c, (e_gpu, e_ref, ratio) in zip(sel, rows):
            _record("dropin_biquad", "%s/%s/ch%d" % (name, how, c), err_gpu=e_gpu, err_ref64=e_ref, ratio=ratio)
            assert e_ref <= REF_TRUTH, (name, how, c, e_ref)   # the table reads the arguments as the reference does
    elif kind == "riir":
        errs = [nerr(y[:, c], want[:, c])[0] for c in sel]
        _record("dropin_riir", "%s/%s" % (name, how), nerr=max(errs))
        assert max(errs) <= TOL, (name, how, errs)
    elif kind == "exact":
        _record("dropin_exact", "%s/%s" % (name, how), equal=bool(np.array_equal(y, want)))
        assert np.array_equal(y, want), (name, how, float(np.max(np.abs(y - want))))
    else:
        e = nerr(y, want)[0]
        _record("dropin_near", "%s/%s" % (name, how), nerr=e)
        assert e <= case["tol"], (name, how, e)


@pytest.mark.parametrize("name", list(CASES))
def test_dropin_effect_forms(libs, name):
    """One chain string through the drop-in and the pure reference, three passes each (module docstring)."""
    case = CASES[name]
    ref, fs = libs, case["fs"]
    x = _input(case)
    truth = coefs = None
    if case["kind"] == "bq":
        coefs = _coefs(ref, case)
        truth = biquad_truth(x, coefs)
    for how in ("1024", "4096", "ragged"):
        g = ref.RefChain(case["chain"], fs, C, lib_path=DROPIN)
        r = ref.RefChain(case["chain"], fs, C, lib_path=REFLIB)
        fx_g, fx_r = g.effect_names(), r.effect_names()
        assert fx_g == (case["fx"] if case["fx"] is not None else fx_r), (name, fx_g, fx_r)
        assert g.fs_out == r.fs_out, (name, g.fs_out, r.fs_out)
        assert g.delay() == r.delay(), (name, g.delay(), r.delay())
        d = int(round(r.delay() * fs))     # latency the chain reports and does not align away (biquad -r's blocks)
        y, counts = _pass(g, x, how)
        want, wcounts = _pass(r, x, how)
        g.close()
        r.close()
        assert counts == wcounts, (name, how, counts, wcounts)
        assert y.shape == want.shape, (name, how, y.shape, want.shape)
        if r.fs_out == fs:
            # unselected channels: the input, delayed by the chain's latency, then the drain's silence
            assert y.shape[0] >= N + d, (name, how, y.shape)
            for c in range(C):
                if c not in case["touched"]:
                    assert np.array_equal(y[d:d + N, c], x[:, c]), (name, how, c)
                    assert not np.any(y[:d, c]) and not np.any(y[d + N:, c]), (name, how, c)
        _check_values(name, case, how, y, want, x, truth, coefs)


def test_dropin_same_rate_resample_is_dropped(libs):
    """`resample` to the stream's own rate returns an effect without run(), which both chains drop."""
    for spec in ("resample 48000", "resample 48k", "resample x1", "resample /1", "eq 1k 1.0 3 resample 48k"):
        names = [libs.RefChain(spec, 48000, C, lib_path=p).effect_names() for p in (DROPIN, REFLIB)]
        assert names[0] == names[1] and "resample" not in names[0], (spec, names)


@pytest.mark.parametrize("name", list(REFUSALS))
def test_dropin_refusals(libs, name):
    """Both libraries refuse the chain: the reference check named in the table, and the shim's copy of it."""
    chain, fs, why, run_ref = REFUSALS[name]
    paths = (DROPIN, REFLIB) if run_ref else (DROPIN,)
    for p in paths:
        with pytest.raises(ValueError):
            libs.RefChain(chain, fs, C, lib_path=p)


@pytest.mark.parametrize("name", list(CASES) + ["refuse/" + n for n in REFUSALS])
def test_python_mirror(libs, name):
    """dsp_b200.effects.build_chain reads every form it supports as the drop-in does (same frame counts, values
    within the case's bounds), raises ChainSyntaxError or NotImplementedError on the forms it leaves to the C shim,
    and refuses what the reference refuses."""
    from dsp_b200.effects import ChainSyntaxError, build_chain
    if name.startswith("refuse/"):
        chain, fs, _, _ = REFUSALS[name[len("refuse/"):]]
        with pytest.raises((ChainSyntaxError, NotImplementedError)):
            build_chain(chain, fs, C)
        return
    case = CASES[name]
    if not case["mirror"]:
        with pytest.raises((ChainSyntaxError, NotImplementedError)):
            build_chain(case["chain"], case["fs"], C)
        return
    x = _input(case)
    ec = build_chain(case["chain"], case["fs"], C)
    y, counts = ec.process(x, 1024)
    ec.close()
    g = libs.RefChain(case["chain"], case["fs"], C, lib_path=DROPIN)
    want, wcounts = _pass(g, x, "1024")
    g.close()
    assert ec.fs_out == g.fs_out
    assert counts == wcounts, (name, counts, wcounts)
    assert y.shape == want.shape
    if case["kind"] == "bq":
        coefs = _coefs(libs, case)
        sel = case["touched"]
        for c, (e_gpu, e_ref, ratio) in zip(sel, biquad_within_ref(y[:, sel], x[:, sel], coefs[:, sel])):
            _record("mirror_biquad", "%s/ch%d" % (name, c), err_gpu=e_gpu, err_ref64=e_ref, ratio=ratio)
    else:
        # the mirror builds the same operators in the same order as the drop-in's device chain
        assert np.array_equal(y, want), (name, float(np.max(np.abs(y - want))))


def test_absorb_after_run_keeps_both_cascades_state(gpu_lib):
    """dspb200_chain_absorb fuses neighbouring cascades into one operator only while neither has run since its last
    reset(); a fused operator starts from zero state.  Absorbing after 5000 frames must continue both cascades:
    the stream equals the un-absorbed pair bit for bit.  Fresh chains, and chains reset after running, still fuse."""
    from oracle import restate
    fs = 48000
    ca = np.array([gpu_lib.biquad_design(13, fs, 100.0, 0.7, 6.0), gpu_lib.biquad_design(8, fs, 30.0, 0.5)])
    cb = np.array([gpu_lib.biquad_design(7, fs, 200.0, 2.0), gpu_lib.biquad_design(14, fs, 300.0, 0.7, -4.0)])
    x = bq_inputs(fs, 12000, seed=5)
    cuts = [0, 1000, 5000, 6024, 9000, 12000]
    a0, b0 = gpu_lib.Chain(fs, C).add_biquad(ca), gpu_lib.Chain(fs, C).add_biquad(cb)
    want = np.concatenate([b0.run(a0.run(x[p:q]).copy()).copy() for p, q in zip(cuts[:-1], cuts[1:])])
    a, b = gpu_lib.Chain(fs, C).add_biquad(ca), gpu_lib.Chain(fs, C).add_biquad(cb)
    got = [b.run(a.run(x[p:q]).copy()).copy() for p, q in zip(cuts[:2], cuts[1:3])]
    a.absorb(b)
    assert a.n_ops == 2, a.describe()          # ran: appended, not fused
    got += [a.run(x[p:q]).copy() for p, q in zip(cuts[2:-1], cuts[3:])]
    got = np.concatenate(got)
    assert np.array_equal(got, want), float(np.max(np.abs(got - want)))
    for ch in (a0, b0, a, b):
        ch.close()
    # fresh chains fuse into one operator, and so do chains reset after running; that one runs the whole cascade
    f, g = gpu_lib.Chain(fs, C).add_biquad(ca), gpu_lib.Chain(fs, C).add_biquad(cb)
    f.absorb(g)
    assert f.n_ops == 1, f.describe()
    f.close()
    g.close()
    f, g = gpu_lib.Chain(fs, C).add_biquad(ca), gpu_lib.Chain(fs, C).add_biquad(cb)
    f.run(x[:3000])
    g.run(x[:3000])
    f.reset()
    g.reset()
    f.absorb(g)
    assert f.n_ops == 1, f.describe()
    y = np.concatenate([f.run(x[p:p + 4096]).copy() for p in range(0, x.shape[0], 4096)])
    f.close()
    g.close()
    both = np.concatenate([ca, cb])
    assert nerr(y, restate.biquad_cascade(x, both))[0] <= 1e-12
