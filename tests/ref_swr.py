"""libswresample as the ffmpeg command line runs it, for the tests: the `-ac 1 -ar <rate> -acodec pcm_s16le` conversion
of the reference's demuxing call, driven through ctypes on the libswresample the opencv-python wheel ships beside the
libraries oracle/ref_flac.py loads (libswresample 6).

    convert(pcm, layout, in_rate, out_rate, path='fma3')  S16 interleaved (frames, channels) -> S16 mono at out_rate,
                                                          fed in decoder-sized chunks, then flushed
    matrix(layout)                                        swr_build_matrix2's mono row with the defaults
    float_bank(in_rate, out_rate)                         the float filter bank, read out by impulses
    defaults()                                            the option defaults the resampler is built from

`path` picks the CPU path through av_force_cpu_flags: 'fma3' (what ffmpeg runs on an x86-64 CPU with AVX2 and FMA3),
'avx', 'sse' or 'c'.  The setting is process wide, so every call restores automatic detection (-1) when it ends.  The
'fma3' and 'avx' paths need a CPU that has those instructions; they are checked in /proc/cpuinfo first so that a
missing instruction set fails with a message instead of an illegal instruction.
Test infrastructure only: the product never imports this."""
import ctypes
import glob
import os

import numpy as np

from oracle import ref_flac

AV_SAMPLE_FMT_S16, AV_SAMPLE_FMT_FLT, AV_SAMPLE_FMT_S16P, AV_SAMPLE_FMT_FLTP = 1, 3, 6, 8
AV_CHANNEL_ORDER_NATIVE = 1
AV_CH_FRONT_CENTER = 0x4
_SSE = 0x1 | 0x2 | 0x8 | 0x10 | 0x40 | 0x80 | 0x100 | 0x200 | 0x1000    # MMX .. SSE4.2, CMOV
PATHS = {'c': 0, 'sse': _SSE, 'avx': _SSE | 0x4000, 'fma3': _SSE | 0x4000 | 0x10000}
_NEEDS = {'c': (), 'sse': ('sse4_2',), 'avx': ('sse4_2', 'avx'), 'fma3': ('sse4_2', 'avx', 'fma')}
_lib = None


class ChLayout(ctypes.Structure):
    _fields_ = [('order', ctypes.c_int), ('nb_channels', ctypes.c_int), ('mask', ctypes.c_uint64),
                ('opaque', ctypes.c_void_p)]


def layout(mask):
    return ChLayout(AV_CHANNEL_ORDER_NATIVE, bin(mask).count('1'), mask, None)


def lib():
    global _lib
    if _lib is not None:
        return _lib
    _, _, util = ref_flac.libs()
    import cv2
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(cv2.__file__))), 'opencv_python_headless.libs')
    hits = sorted(glob.glob(os.path.join(d, 'libswresample-*.so*')))
    if not hits:
        raise RuntimeError('libswresample not found in %s' % d)
    swr = ctypes.CDLL(hits[0], mode=ctypes.RTLD_GLOBAL)
    vp, i32, lp = ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ChLayout)
    swr.swr_alloc_set_opts2.argtypes = [ctypes.POINTER(vp), lp, i32, i32, lp, i32, i32, i32, vp]
    swr.swr_alloc_set_opts2.restype = i32
    swr.swr_init.argtypes = [vp]
    swr.swr_init.restype = i32
    swr.swr_convert.argtypes = [vp, ctypes.POINTER(vp), i32, ctypes.POINTER(vp), i32]
    swr.swr_convert.restype = i32
    swr.swr_free.argtypes = [ctypes.POINTER(vp)]
    swr.swr_build_matrix2.argtypes = [lp, lp, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                      ctypes.c_double, ctypes.POINTER(ctypes.c_double), ctypes.c_ssize_t, i32, vp]
    swr.swr_build_matrix2.restype = i32
    util.av_force_cpu_flags.argtypes = [i32]
    util.av_opt_set_int.argtypes = [vp, ctypes.c_char_p, ctypes.c_int64, i32]
    util.av_opt_set_int.restype = i32
    util.av_opt_get_int.argtypes = [vp, ctypes.c_char_p, i32, ctypes.POINTER(ctypes.c_int64)]
    util.av_opt_get_int.restype = i32
    util.av_opt_get_double.argtypes = [vp, ctypes.c_char_p, i32, ctypes.POINTER(ctypes.c_double)]
    util.av_opt_get_double.restype = i32
    _lib = (swr, util)
    return _lib


def _check_cpu(path):
    with open('/proc/cpuinfo') as f:
        flags = next((line.split(':', 1)[1].split() for line in f if line.startswith('flags')), [])
    missing = [n for n in _NEEDS[path] if n not in flags]
    if missing:
        raise RuntimeError("ref_swr: the '%s' path needs a CPU with %s; this one lacks %s"
                           % (path, ', '.join(_NEEDS[path]), ', '.join(missing)))


def _context(in_mask, in_fmt, in_rate, out_mask, out_fmt, out_rate, options=()):
    swr, util = lib()
    s = ctypes.c_void_p()
    lin, lout = layout(in_mask), layout(out_mask)
    rc = swr.swr_alloc_set_opts2(ctypes.byref(s), ctypes.byref(lout), out_fmt, out_rate, ctypes.byref(lin), in_fmt,
                                 in_rate, 0, None)
    assert rc >= 0 and s, 'swr_alloc_set_opts2: %d' % rc
    for name, value in options:
        assert util.av_opt_set_int(s, name.encode(), value, 0) >= 0, name
    return s


def _run(s, planes_in, n_in, out_dtype, out_channels, chunk, bound):
    """swr_init, then swr_convert over `chunk`-frame pieces (None: the whole buffer), each drained by calls with no new
    input while they fill the output, then flush calls until one gives nothing.  At most `bound` frames come out per
    call (libswresample sizes its internal buffers by the call's output room).  planes_in: one contiguous array per
    input plane (packed input: one)."""
    swr, _ = lib()
    rc = swr.swr_init(s)
    assert rc >= 0, 'swr_init: %d' % rc
    cap = bound + 64
    out = np.zeros((cap, out_channels), out_dtype)
    pieces = []
    step = n_in if chunk is None else chunk
    pos = 0
    item = planes_in[0].itemsize * (planes_in[0].shape[1] if planes_in[0].ndim == 2 else 1)

    def call(frames):
        outp = (ctypes.c_void_p * 1)(out.ctypes.data)
        if frames is None:
            got = swr.swr_convert(s, outp, cap, None, 0)
        else:
            inp = (ctypes.c_void_p * len(planes_in))(*[p.ctypes.data + pos * item for p in planes_in])
            got = swr.swr_convert(s, outp, cap, inp, frames)
        assert got >= 0, 'swr_convert: %d' % got
        pieces.append(out[:got].copy())
        return got
    while pos < n_in:
        k = min(step, n_in - pos)
        got = call(k)
        pos += k
        while got == cap:
            got = call(0)
    while call(None) > 0:
        pass
    return np.concatenate(pieces) if pieces else np.zeros((0, out_channels), out_dtype)


class _Flags(object):
    def __init__(self, path):
        if path not in PATHS:
            raise ValueError('path must be one of %s' % sorted(PATHS))
        _check_cpu(path)
        self.path = path

    def __enter__(self):
        lib()[1].av_force_cpu_flags(PATHS[self.path])

    def __exit__(self, *exc):
        lib()[1].av_force_cpu_flags(-1)


def convert(pcm, mask, in_rate, out_rate, path='fma3', chunk=4096, options=()):
    """int16 (frames, channels) interleaved S16 with channel mask `mask` at in_rate -> int16 mono at out_rate, as
    `ffmpeg -ac 1 -ar out_rate -acodec pcm_s16le` writes it (S16 in, S16 out, every other option at its default)."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    if pcm.ndim == 1:
        pcm = pcm[:, None]
    assert pcm.shape[1] == bin(mask).count('1'), 'channel count and layout differ'
    swr, _ = lib()
    with _Flags(path):
        s = _context(mask, AV_SAMPLE_FMT_S16, in_rate, AV_CH_FRONT_CENTER, AV_SAMPLE_FMT_S16, out_rate, options)
        try:
            step = len(pcm) if chunk is None else chunk
            bound = min(len(pcm) + 1024, step + 1024, 1 << 22) * out_rate // in_rate + 4096
            return _run(s, [pcm], len(pcm), np.int16, 1, chunk, bound)[:, 0]
        finally:
            swr.swr_free(ctypes.byref(s))


def convert_float(x, in_rate, out_rate, path='fma3', chunk=None):
    """float32 mono FLT in -> FLT out: the float resampler alone."""
    x = np.ascontiguousarray(x, np.float32)[:, None]
    swr, _ = lib()
    with _Flags(path):
        s = _context(AV_CH_FRONT_CENTER, AV_SAMPLE_FMT_FLT, in_rate, AV_CH_FRONT_CENTER, AV_SAMPLE_FMT_FLT, out_rate)
        try:
            bound = (len(x) + 1024) * out_rate // in_rate + 4096
            return _run(s, [x], len(x), np.float32, 1, chunk, bound)[:, 0]
        finally:
            swr.swr_free(ctypes.byref(s))


def matrix(mask, center=0.7071067811865476, surround=0.7071067811865476, lfe=0.0, maxval=1.0):
    """swr_build_matrix2's row for a mono (front centre) output: one float64 per channel of `mask`, in mask order.
    The defaults are libswresample's (-3 dB centre and surround, LFE muted, normalised to a sum of 1 for integer
    output)."""
    swr, _ = lib()
    m = np.zeros(64 * 64, np.float64)
    rc = swr.swr_build_matrix2(ctypes.byref(layout(mask)), ctypes.byref(layout(AV_CH_FRONT_CENTER)), center, surround,
                               lfe, maxval, 1.0, m.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), 64, 0, None)
    assert rc >= 0, 'swr_build_matrix2: %d' % rc
    return m[:bin(mask).count('1')].copy()


def defaults():
    """{option: value} of a fresh context: the resampler's parameters as ffmpeg builds it."""
    swr, util = lib()
    s = _context(0x3, AV_SAMPLE_FMT_S16, 48000, AV_CH_FRONT_CENTER, AV_SAMPLE_FMT_S16, 12000)
    try:
        out = {}
        for name in ('filter_size', 'phase_shift', 'linear_interp', 'exact_rational', 'filter_type', 'dither_method',
                     'internal_sample_fmt', 'resampler'):
            v = ctypes.c_int64()
            assert util.av_opt_get_int(s, name.encode(), 0, ctypes.byref(v)) >= 0, name
            out[name] = v.value
        for name in ('cutoff', 'kaiser_beta', 'center_mix_level', 'surround_mix_level', 'lfe_mix_level'):
            v = ctypes.c_double()
            assert util.av_opt_get_double(s, name.encode(), 0, ctypes.byref(v)) >= 0, name
            out[name] = v.value
        return out
    finally:
        swr.swr_free(ctypes.byref(s))


def float_bank(in_rate, out_rate, taps, phases, path='fma3'):
    """The float filter bank (phases x taps) of an exact-ratio conversion, read out by impulses of 1.0 on FLT mono:
    every output is then one coefficient times 1.0 plus exact zeros.  Output t reads phase (t * in_g) % out_g at sample
    (t * in_g) // out_g of the stream the resampler sees, whose first (taps - 1) // 2 samples mirror the input's start
    (in_g / out_g: in_rate / out_rate in lowest terms, out_g == phases).  An impulse at input sample k therefore shows
    tap k + (taps - 1) // 2 - sample of that phase; in_g impulse positions cover every tap."""
    import math
    g = math.gcd(in_rate, out_rate)
    in_g, out_g = in_rate // g, out_rate // g
    assert out_g == phases, 'not an exact-ratio bank'
    c = (taps - 1) // 2
    n = 4 * taps + 4 * in_g + 64
    k0 = 2 * taps
    bank = np.full((phases, taps), np.nan, np.float32)
    for j in range(in_g):
        x = np.zeros(n, np.float32)
        x[k0 + j] = 1.0
        y = convert_float(x, in_rate, out_rate, path)
        for t in range(len(y)):
            idx = t * in_g
            p, s = idx % out_g, idx // out_g
            i = k0 + j + c - s
            if 0 <= i < taps and s >= taps:              # far from both mirrored edges
                bank[p, i] = y[t]
    return bank
