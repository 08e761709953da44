"""Python mirror of the reference's effect interface for the hot-path effects.

`build_chain("gain -6 eq 1k 1.0 3 :0,2 fir_p ir.f64 : resample 48k", fs, channels)` accepts the
reference's chain mini-language for the effects this project accelerates -- same names, argument
order and units as `dsp` (effect.c:46-67, biquad.h:97-117, fir.h:30, fir_p.h:30, hilbert.h:28,
resample.h:28, gain.h:33-36) -- and builds ONE device chain (dsp_b200.lib.Chain) from it.
Consecutive biquads are fused into one cascade operator; everything between the single H2D and
the single D2H of a block stays in HBM.

This mirror exists so that parity tests read like runs of the reference CLI.  The drop-in
artefact for the reference's own frontends is the C shim under shim/, not this file.  Host
code that is NOT part of the accelerated path and stays the reference's C in a real deployment
(the chain parser, `align`, drain bookkeeping) is restated here only as far as tests need it.
"""
import importlib
import math
import os
import re

import numpy as np

# the package re-exports a FUNCTION named lib, so fetch the submodule explicitly
_lib = importlib.import_module(".lib", __package__)

BIQUAD_TYPES = {
    # name -> (type number biquad.h:30-52, positional args)
    "lowpass_1": (1, "f"), "highpass_1": (2, "f"), "allpass_1": (3, "f"),
    "lowshelf_1": (4, "fg"), "highshelf_1": (5, "fg"), "lowpass_1p": (6, "f"),
    "lowpass": (7, "fw"), "highpass": (8, "fw"), "bandpass_skirt": (9, "fw"), "bandpass_peak": (10, "fw"),
    "notch": (11, "fw"), "allpass": (12, "fw"), "eq": (13, "fwg"), "lowshelf": (14, "fwg"), "highshelf": (15, "fwg"),
    "lowpass_transform": (16, "fwfw"), "highpass_transform": (17, "fwfw"), "linkwitz_transform": (17, "fwfw"),
}
WIDTH_Q, WIDTH_SLOPE, WIDTH_SLOPE_DB, WIDTH_BW_OCT, WIDTH_BW_HZ = 1, 2, 3, 4, 5
IDENTITY = (1.0, 0.0, 0.0, 0.0, 0.0)


class ChainSyntaxError(ValueError):
    pass


# what strtod() reads: leading white space, a sign, then a decimal number with an optional exponent, a hexadecimal
# one with an optional binary exponent, inf[inity] or nan[(chars)] (no digit separators, unlike Python's float())
_STRTOD = re.compile(r"\s*([+-]?)(?:(?P<dec>(?:[0-9]+\.?[0-9]*|\.[0-9]+)(?:[eE][+-]?[0-9]+)?)"
                     r"|(?P<hex>0[xX](?:[0-9a-fA-F]+\.?[0-9a-fA-F]*|\.[0-9a-fA-F]+)(?:[pP][+-]?[0-9]+)?)"
                     r"|(?P<inf>[iI][nN][fF](?:[iI][nN][iI][tT][yY])?)|(?P<nan>[nN][aA][nN](?:\([0-9A-Za-z_]*\))?))")


def parse_num(s, what="value"):
    """strtod() over the whole word, as the reference's CHECK_ENDPTR demands (util.c:35-47)."""
    m = _STRTOD.fullmatch(s)
    if not m:
        raise ChainSyntaxError("failed to parse %s: %s" % (what, s))
    sign = -1.0 if m.group(1) == "-" else 1.0
    if m.group("dec"):
        return sign * float(m.group("dec"))
    if m.group("hex"):
        h = m.group("hex")
        return sign * float.fromhex(h if "p" in h.lower() else h + "p0")
    return sign * float("inf" if m.group("inf") else "nan")


def parse_int(s, what="value"):
    """strtol(s, 10) over the whole word."""
    if not re.fullmatch(r"\s*[+-]?[0-9]+", s):
        raise ChainSyntaxError("failed to parse %s: %s" % (what, s))
    return int(s)


def parse_freq(s, what="f0"):
    """util.c:49-63: a number, optionally followed by k"""
    if s.endswith("k"):
        return parse_num(s[:-1], what) * 1000.0
    return parse_num(s, what)


def parse_width(s):
    """biquad.c:27-89 -> (width, width_type)"""
    if s.startswith("bw") and len(s) > 2:
        m = re.fullmatch(r"(\s*[+-]?[0-9]+)(?:\.(\s*[+-]?[0-9]+))?", s[2:])
        if not m:
            raise ChainSyntaxError("failed to parse width: %s" % s)
        order = int(m.group(1))
        if order < 2:
            raise ChainSyntaxError("filter order must be >= 2")
        n_biquads = order // 2
        p_idx = int(m.group(2)) if m.group(2) is not None else 0
        if p_idx < 0 or p_idx >= n_biquads:
            raise ChainSyntaxError("filter index out of range")
        p_idx = n_biquads - p_idx
        return 1.0 / (2.0 * math.sin(math.pi / order * (p_idx - 0.5))), WIDTH_Q
    suffix = {"q": WIDTH_Q, "s": WIDTH_SLOPE, "d": WIDTH_SLOPE_DB, "o": WIDTH_BW_OCT, "h": WIDTH_BW_HZ, "k": WIDTH_BW_HZ}
    if s and s[-1] in suffix:
        w = parse_num(s[:-1], "width")
        if s[-1] == "k":
            w *= 1000.0
        return w, suffix[s[-1]]
    return parse_num(s, "width"), WIDTH_Q


def parse_selector(s, n):
    """util.c:131-188: "0,2", "1-3", "-2", "3-", "" or "-" = all."""
    sel = [0] * n
    if s in ("", "-"):
        return [1] * n
    for part in s.split(","):
        if "-" in part:
            a, _, b = part.partition("-")
            lo = int(a) if a else 0
            hi = int(b) if b else n - 1
        else:
            lo = hi = int(part)
        if lo < 0 or hi > n - 1 or hi < lo:
            raise ChainSyntaxError("selector out of range: %r" % s)
        for k in range(lo, hi + 1):
            sel[k] = 1
    return sel


def _read_filter(args, fs, n_sel, dir_):
    """fir_util.c:25-185 for the input forms the tests use: `coefs:a,b,c/d,e,f` and raw float64 PCM
    (`-t pcm -e double [-c N] [-r fs] path`).  Returns taps [frames, filter_channels]."""
    opts = {"c": None}
    i = 0
    while i < len(args) and args[i].startswith("-") and len(args[i]) == 2 and args[i][1] in "tecrBLNa":
        if args[i][1] in "BLN":
            i += 1
            continue
        opts[args[i][1]] = args[i + 1]
        i += 2
    rest = args[i:]
    if len(rest) == 2:
        max_part = int(rest[0])     # fir_p's optional max_part_len: a CPU latency knob, irrelevant here
        del max_part
        rest = rest[1:]
    if len(rest) != 1:
        raise ChainSyntaxError("fir: expected one filter argument")
    path = rest[0]
    if "a" in opts:
        raise NotImplementedError("-a alignment offsets are handled by the C shim (fir_util.c:187-205)")
    if path.startswith("coefs:"):
        cols = [[float(v) for v in col.split(",")] for col in path[len("coefs:"):].split("/")]
        frames = max(len(c) for c in cols)
        taps = np.zeros((frames, len(cols)))
        for k, c in enumerate(cols):
            taps[:len(c), k] = c
        return taps
    if opts.get("t", "pcm") != "pcm" or opts.get("e", "double") not in ("double", "f64", "float64"):
        raise NotImplementedError("filter files other than raw float64 PCM go through the reference codec layer")
    fc = int(opts["c"]) if opts["c"] else n_sel      # fir_util.c:131: default channels = stream channels
    if "r" in opts and opts["r"] is not None and int(parse_freq(opts["r"])) != fs:
        raise ChainSyntaxError("filter sample rate mismatch")
    data = np.fromfile(os.path.join(dir_ or ".", path), dtype="<f8")
    return data[:(data.shape[0] // fc) * fc].reshape(-1, fc)


def _next_fast_len(n):
    while True:
        m = n
        for p in (2, 3, 5, 7):
            while m % p == 0:
                m //= p
        if m == 1:
            return n
        n += 1


class EffectsChain:
    """What a frontend sees: run()/drain() over host blocks (effects_chain.h:47,52)."""

    def __init__(self, fs, channels, devices=None, slabs_per_device=1, block_hint=0):
        self.fs_in = fs
        self.channels = channels
        self.chain = _lib.Chain(fs, channels, devices, slabs_per_device)
        self.block_hint = block_hint
        self.names = []
        self._pending_biquads = []          # [stage][channel] -> c5
        self._drain = [0] * channels         # cumulative drain samples per channel (effects_chain.c:877-923)
        self._fs = fs
        self._align_discard = 0             # fir latency to discard at the tail (align.c:53-62)
        self._align_delay_sel = None
        self._discarded = 0
        self._delay_buf = None
        self.drain_frames = 0

    # -- builders ------------------------------------------------------------------------
    def _flush_biquads(self):
        if self._pending_biquads:
            self.chain.add_biquad(np.array(self._pending_biquads, dtype=np.float64))
            self._pending_biquads = []

    def add_effect(self, name, args, sel, dir_=None):
        C = self.channels
        if name in BIQUAD_TYPES or name in ("biquad", "deemph"):
            c5 = self._design(name, args)
            self._pending_biquads.append([tuple(c5) if sel[k] else IDENTITY for k in range(C)])
            self.names.append(name)
            return
        self._flush_biquads()
        if name in ("gain", "mult", "add"):
            if len(args) != 1:
                raise ChainSyntaxError("%s: usage: %s value" % (name, name))
            v = parse_num(args[0], name)
            if name == "gain":
                v = 10.0 ** (v / 20.0)
            if name == "add":
                self.chain.add_gain(np.ones(C), np.array([v if sel[k] else 0.0 for k in range(C)]))
            else:
                self.chain.add_gain(np.array([v if sel[k] else 1.0 for k in range(C)]))
        elif name in ("fir", "fir_p"):
            n_sel = sum(sel)
            taps = _read_filter(args, self._fs, n_sel, dir_)
            self._add_fir(name, taps, sel)
        elif name == "hilbert":
            conv, do_align, angle = "fir", False, -math.pi / 2
            a = list(args)
            # dsp_getopt(argc - 1, "pzca:") (hilbert.c:36-54): options only in front of the last word
            while len(a) > 1 and a[0].startswith("-") and len(a[0]) > 1:
                o = a.pop(0)
                for i, ch in enumerate(o[1:]):
                    if ch == "p" or ch == "z":
                        conv = "fir_p"
                    elif ch == "c":
                        do_align = True
                    elif ch == "a":
                        if o[i + 2:]:
                            v = o[i + 2:]
                        elif len(a) > 1:
                            v = a.pop(0)
                        else:
                            raise ChainSyntaxError("hilbert: option -a needs an angle")
                        angle = parse_num(v, "angle") / 180.0 * math.pi
                        break
                    else:
                        raise ChainSyntaxError("hilbert: unknown option -%s" % ch)
            if len(a) != 1:
                raise ChainSyntaxError("hilbert: usage: hilbert [-p|-z] [-c] [-a angle] taps")
            n_taps = parse_int(a[0], "taps")
            if n_taps <= 3 or n_taps % 2 == 0:
                raise ChainSyntaxError("hilbert: taps must be > 3 and odd")
            if do_align:
                raise NotImplementedError("hilbert -c needs the reference's align pass (C shim)")
            taps = _lib.hilbert_taps(n_taps, angle)
            self._add_fir(conv, taps[:, None], sel)
        elif name == "resample":
            if len(args) not in (1, 2):
                raise ChainSyntaxError("resample: usage: resample [bandwidth] fs")
            bw = parse_num(args[0], "bandwidth") if len(args) == 2 else 0.0
            if len(args) == 2 and not 0.7 <= bw <= 0.999:
                raise ChainSyntaxError("resample: bandwidth out of range: %s" % args[0])
            r = args[-1]
            if r.startswith("x"):
                rate = self._fs * parse_int(r[1:], "fs multiplier")
            elif r.startswith("/"):
                div = parse_int(r[1:], "fs divisor")
                if div == 0 or self._fs % div:
                    raise ChainSyntaxError("resample: %d is not a factor of %d" % (div, self._fs))
                rate = self._fs // div
            else:
                f = parse_freq(r, "fs")
                rate = int(math.floor(abs(f) + 0.5)) * (1 if f >= 0 else -1)    # lround()
            if rate <= 0:
                raise ChainSyntaxError("resample: rate out of range: %s" % r)
            if self._align_discard:
                raise NotImplementedError("fir latency followed by a rate change needs the reference's align pass")
            if rate != self._fs:
                g = math.gcd(rate, self._fs)
                n, d = rate // g, self._fs // g
                self.chain.add_resample(rate, bw)
                self._drain = [(s * n + d - 1) // d for s in self._drain]
                self._fs = rate
        else:
            raise ChainSyntaxError("effect %r is not on the accelerated path" % name)
        self.names.append(name)

    def _add_fir(self, name, taps, sel):
        frames = taps.shape[0]
        latency = 0
        # fir.c:240 (<= 16 taps: direct), fir_p.c:364-365 (<= 32 taps: fir direct), else fir = FFT with latency len
        if name == "fir" and frames > 16:
            latency = _next_fast_len(frames)
            if self._align_discard:
                raise NotImplementedError("two latent fir effects need the reference's align pass")
            self._align_discard = latency
            self._align_delay_sel = list(sel)
        self.chain.add_fir(taps, selector=sel, latency=latency, block_hint=self.block_hint)
        for k in range(self.channels):
            if sel[k]:
                self._drain[k] += latency + frames - 1

    def _design(self, name, args):
        fs = self._fs
        if args and args[0].startswith("-r"):
            raise NotImplementedError("biquad -r (reverse IIR) is designed by the reference (C shim)")
        if name == "biquad":
            if len(args) != 6:
                raise ChainSyntaxError("biquad: expected 6 arguments")
            b0, b1, b2, a0, a1, a2 = (parse_num(v, "coefficient") for v in args)
            return (b0 / a0, b1 / a0, b2 / a0, a1 / a0, a2 / a0)
        if name == "deemph":
            if args:
                raise ChainSyntaxError("deemph: expected no arguments")
            preset = {44100: (5283, 0.4845, -9.477), 48000: (5356, 0.479, -9.62)}.get(fs)
            if not preset:
                raise ChainSyntaxError("deemph: sample rate must be 44100 or 48000")
            return _lib.biquad_design(15, fs, preset[0], preset[1], preset[2], 0.0, WIDTH_SLOPE)
        type_, sig = BIQUAD_TYPES[name]
        if len(args) != len(sig):
            raise ChainSyntaxError("%s: expected %d arguments" % (name, len(sig)))
        wt = WIDTH_Q
        vals = []
        for kind, a in zip(sig, args):
            if kind == "f":
                f = parse_freq(a)
                if not 0.0 <= f < fs / 2.0:       # CHECK_FREQ (util.h:36-37)
                    raise ChainSyntaxError("%s: frequency out of range: %s" % (name, a))
                vals.append(f)
            elif kind == "w":
                w, wt = parse_width(a)
                if not w > 0.0:
                    raise ChainSyntaxError("%s: width out of range: %s" % (name, a))
                # biquad.c:476,484,492,495: slope widths only on the shelves, only Q on the transforms
                if wt in (WIDTH_SLOPE, WIDTH_SLOPE_DB) and name not in ("lowshelf", "highshelf"):
                    raise ChainSyntaxError("%s: invalid width type: %s" % (name, a))
                if sig == "fwfw" and wt != WIDTH_Q:
                    raise ChainSyntaxError("%s: invalid width type: %s" % (name, a))
                vals.append(w)
            else:
                vals.append(parse_num(a, "gain"))
        if sig == "f":
            arg = (vals[0], 0.0, 0.0, 0.0)
        elif sig == "fg":
            arg = (vals[0], 0.0, vals[1], 0.0)
        elif sig == "fw":
            arg = (vals[0], vals[1], 0.0, 0.0)
        elif sig == "fwg":
            arg = (vals[0], vals[1], vals[2], 0.0)
        else:
            arg = tuple(vals)
        return _lib.biquad_design(type_, fs, arg[0], arg[1], arg[2], arg[3], wt)

    def finish(self):
        self._flush_biquads()
        g = math.gcd(self.fs_in, self._fs)
        self.drain_frames = max(self._drain) * (self.fs_in // g) // (self._fs // g) if self._drain else 0
        self.fs_out = self._fs
        if self._align_discard:
            # unselected channels are delayed by the same latency (align.c:35-44,130-153)
            self._delay_buf = np.zeros((self._align_discard, self.channels))
        return self

    # -- running -------------------------------------------------------------------------
    def _align(self, y):
        if not self._align_discard or y.shape[0] == 0:
            return y
        L = self._align_discard
        sel = self._align_delay_sel
        idx = [k for k in range(self.channels) if not sel[k]]
        if idx:
            joined = np.concatenate([self._delay_buf[:, idx], y[:, idx]], axis=0)
            y = y.copy()
            y[:, idx] = joined[:y.shape[0]]
            self._delay_buf[:, idx] = joined[-L:]
        if self._discarded < L:
            drop = min(L - self._discarded, y.shape[0])
            self._discarded += drop
            y = y[drop:]
        return y

    def run(self, x):
        return self._align(self.chain.run(x).copy())

    def process(self, x, block):
        outs, counts = [], []
        for i in range(0, x.shape[0], block):
            y = self.run(x[i:i + block])
            outs.append(y)
            counts.append(y.shape[0])
        left = self.drain_frames
        while left > 0:
            f = min(block, left)
            left -= f
            y = self.run(np.zeros((f, self.channels)))
            outs.append(y)
            counts.append(y.shape[0])
        while True:
            y = self.chain.drain(block)
            if y is None:
                break
            outs.append(y)
            counts.append(y.shape[0])
        return (np.concatenate(outs, axis=0) if outs else np.zeros((0, self.channels))), counts

    def reset(self):
        self.chain.reset()
        self._discarded = 0
        if self._delay_buf is not None:
            self._delay_buf[:] = 0.0

    def close(self):
        self.chain.close()


def build_chain(chain_str, fs, channels, dir=None, devices=None, slabs_per_device=1, block_hint=0):
    """effects_chain.c:445-603 for the subset: `:selector` tokens and effect words."""
    ec = EffectsChain(fs, channels, devices, slabs_per_device, block_hint)
    sel = [1] * channels
    words = chain_str.split()
    known = set(BIQUAD_TYPES) | {"biquad", "deemph", "gain", "mult", "add", "fir", "fir_p", "hilbert", "resample"}
    i = 0
    try:
        while i < len(words):
            w = words[i]
            if w.startswith(":"):
                sel = parse_selector(w[1:], channels)
                i += 1
                continue
            if w not in known:
                raise ChainSyntaxError("unknown or unaccelerated effect: %r" % w)
            j = i + 1
            while j < len(words) and not words[j].startswith(":") and words[j] not in known:
                j += 1
            ec.add_effect(w, words[i + 1:j], sel, dir)
            i = j
        return ec.finish()
    except BaseException:
        ec.close()          # a refused chain frees its device chain now, not when the collector finds it
        raise
