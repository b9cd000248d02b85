"""Drop-in replacement for the reference's audio stream class (reference wav.py:104-188).

Same constructor, attributes and methods as the reference ``WavStream`` so that
``sushi.py``'s ``calculate_shifts`` (sushi.py:400-508) runs unchanged on top of it:

    WavStream(path, sample_rate=12000, sample_type='uint8')        wav.py:108
    .data .sample_rate .sample_count .padding_size .duration_seconds
    .get_substream(start, end)                  -> ndarray view     wav.py:168-171
    .find_substream(pattern, center, window)    -> (np.float32, float)   wav.py:177-188

The arithmetic of find_substream -- OpenCV's matchTemplate(TM_SQDIFF_NORMED) and
the argmin -- runs on the GPU behind the C ABI in include/sushi_b200.h.  All time ->
sample conversions stay here, in Python, written exactly as the reference writes
them, so the integer offsets handed to the library are bit-identical.
"""
import ctypes
import logging
import math
from time import time
import weakref

import numpy as np

from . import _native, swr
from ._nvtx import nvtx_range
from .common import SushiError, clip, py2_round
from .inputs import open_input, FlacFile, is_flac   # noqa: F401  (the FLAC reader stays importable from here)
from .wav import DownmixedWavFile, decode_downmix, nearest_index_map, normalise_host   # noqa: F401

_DTYPES = {'uint8': (np.uint8, _native.SB_U8), 'float32': (np.float32, _native.SB_F32)}

# live streams, so that a pattern that is a *view* of some stream's .data (what
# get_substream / np.split return, sushi.py:417,445) is recognised and handed to the
# GPU as an (offset, length) descriptor instead of being uploaded again.
_live_streams = weakref.WeakSet()


class StreamGeometry(object):
    """What the time -> sample arithmetic of the reference needs to know about a stream (wav.py:164-184):
    rate, padding, sample count and the length of the padded array.  WavStream derives from it; the
    multi-GPU path plans every rank's queries from these four numbers alone (sushi_b200/parallel.py)."""
    PADDING_SECONDS = 10

    def __init__(self, sample_rate, padding_size, sample_count, total_samples):
        self.sample_rate, self.padding_size, self.sample_count = sample_rate, int(padding_size), sample_count
        self._total = int(total_samples)

    @property
    def total_samples(self):
        data = getattr(self, 'data', None)
        return data.shape[1] if data is not None else self._total

    @property
    def duration_seconds(self):
        return self.sample_count / self.sample_rate

    def _get_sample_for_time(self, timestamp):
        # REAL sample for a time, padding included (wav.py:173-175); int() truncates toward zero
        return int(self.sample_rate * timestamp) + self.padding_size

    def plan_queries(self, src_stream, starts, ends, centers, windows):
        """Integer descriptors of many find_substream calls at once.

        Query q searches src_stream.get_substream(starts[q], ends[q]) in this stream around
        centers[q] +- windows[q].  Returns (tmpl_off, tmpl_len, lag0, nlags, start_times) as
        int64/float64 arrays.  Vectorised, but operation for operation the scalar code of
        get_substream / find_substream (wav.py:168-184): float64 product, truncation toward zero,
        min-then-max clipping, NumPy slice clamping -- so the integers are identical
        (tests/test_host_logic.py checks this against the scalar path).
        """
        starts = np.asarray(starts, np.float64); ends = np.asarray(ends, np.float64)
        centers = np.asarray(centers, np.float64); windows = np.asarray(windows, np.float64)

        def sample_for_time(stream, t):                       # wav.py:173-175
            return np.trunc(stream.sample_rate * t).astype(np.int64) + stream.padding_size

        def slice_bounds(lo, hi, total):                      # what data[:, lo:hi] resolves to
            lo = np.where(lo < 0, np.maximum(lo + total, 0), np.minimum(lo, total))
            hi = np.where(hi < 0, np.maximum(hi + total, 0), np.minimum(hi, total))
            return lo, np.maximum(hi - lo, 0)

        toff, tlen = slice_bounds(sample_for_time(src_stream, starts), sample_for_time(src_stream, ends),
                                  src_stream.total_samples)
        dur = self.duration_seconds
        t0 = np.maximum(np.minimum(centers - windows, dur), -self.PADDING_SECONDS)           # wav.py:178
        t1 = np.maximum(np.minimum(centers + windows, dur + self.PADDING_SECONDS), 0)        # wav.py:179
        lag0, span = slice_bounds(sample_for_time(self, t0), sample_for_time(self, t1) + tlen, self.total_samples)
        bad = np.nonzero((tlen < 1) | (span < tlen))[0]
        if len(bad):
            q = int(bad[0])
            raise SushiError('query {0}: pattern of {1} samples does not fit its search span of {2}'.format(
                q, int(tlen[q]), int(span[q])))
        return toff, tlen, lag0, span - tlen + 1, t0


class WavStream(StreamGeometry):
    READ_CHUNK_SIZE = 1  # seconds per resample chunk (wav.py:105)

    def __init__(self, path, sample_rate=12000, sample_type='uint8', device=None, loader='gpu', track=None,
                 ffmpeg_audio=False):
        """loader='gpu' (default): decode / resample / pad / normalise on the GPU (sb_load_pcm +
        sb_normalise); loader='host' runs the NumPy mirror of the same arithmetic and uploads the
        result (kept as the cross-check; both give bit-identical .data).  `path` is a file of any format in
        inputs.READERS, or an opened MatroskaFile, Mp4File or TransportStream (left open; a MatroskaFile's frames then
        come from one walk shared with the script and timecodes).  A container loads its audio stream `track` (a stream
        id; None: the only audio track, else the default one, as the reference selects).  ffmpeg_audio=True loads an
        input that is not a RIFF WAV file as the mono `sample_rate` WAV the reference's ffmpeg call writes for it
        (sushi_b200/swr.py); a WAV file loads as it always does."""
        if sample_type not in _DTYPES:
            raise SushiError('Unknown sample type of WAV stream, must be uint8 or float32')
        self._handle = None
        before_read = time()
        reader, name = open_input(path)
        try:
            audio = reader.select_audio(track)
            if ffmpeg_audio and name != 'WAV':
                self._load_ffmpeg(audio, sample_rate, sample_type, device, loader)
            elif audio.label is None:
                self._load_pcm(audio.pcm, sample_rate, sample_type, device, loader)
            else:
                # compressed inputs are decoded on the GPU only
                if loader != 'gpu':
                    raise SushiError("{0}: {1} input needs loader='gpu' (there is no host {1} decoder)".format(
                        audio.path, audio.label))
                self._load_decoded(audio.decode(device), sample_rate, sample_type, device, audio.check)
        except Exception as e:
            if isinstance(e, SushiError) or name != 'WAV':
                raise
            raise SushiError('Error while loading {0}: {1}'.format(path, e))        # as the reference does (wav.py:158-159)
        finally:
            if reader is not path and hasattr(reader, 'close'):
                reader.close()
        logging.info('Done reading {0} {1} in {2}s'.format(name, path, time() - before_read))

    def _load_pcm(self, pcm, sample_rate, sample_type, device, loader):
        """Integer PCM as a reader lays it out, pcm() -> (bytes, frames, channels, sample width, rate, big-endian):
        sb_load_pcm (little-endian), sb_pcm_from_be (big-endian) or, for loader='host', the host loader."""
        data, frames, channels, width, rate, big = pcm()
        if loader != 'gpu':
            if big:
                data = np.frombuffer(data, np.uint8).reshape(-1, width)[:, ::-1].tobytes()
            self._load(DownmixedWavFile.from_bytes(data, channels, rate, width, frames), sample_rate, sample_type)
            self._upload(device)
        elif big:
            buf = np.frombuffer(data, dtype=np.uint8)
            h = _native.decode(device, 'sb_pcm_from_be', buf.ctypes.data_as(ctypes.c_void_p), frames, channels, width,
                               rate)
            self._load_decoded(h, sample_rate, sample_type, device)
        else:
            self._load_gpu(data, frames, channels, width, rate, sample_rate, sample_type, device)

    def _load_ffmpeg(self, audio, sample_rate, sample_type, device, loader):
        """ffmpeg_audio=True: the reader's audio decoded (or container PCM uploaded) to an sb_pcm, converted by
        sb_pcm_swr to the ffmpeg command line's mono `sample_rate` samples and loaded as their WAV loads."""
        swr.check(audio)
        if loader != 'gpu':
            raise SushiError("{0}: --ffmpeg-audio needs loader='gpu'".format(audio.path))
        if audio.label is None:
            data, frames, channels, width, rate, big = audio.pcm()
            buf = np.frombuffer(data, dtype=np.uint8)
            h = _native.decode(device, 'sb_pcm_from_be' if big else 'sb_pcm_from_le',
                               buf.ctypes.data_as(ctypes.c_void_p), frames, channels, width, rate)
        else:
            h = audio.decode(device)
        self._load_decoded(swr.convert(device, h, audio, sample_rate), sample_rate, sample_type, device)

    def _load_decoded(self, h, sample_rate, sample_type, device, check=None):
        """_load_gpu_with on a decoder's sb_pcm handle `h` (sb_pcm_load), which it destroys; check(frames) may refuse
        the decoded frame count first."""
        lib = _native.lib(device)
        try:
            frames, channels, rate = ctypes.c_int64(), ctypes.c_int32(), ctypes.c_int32()
            _native.check(lib.sb_pcm_info(h, ctypes.byref(frames), ctypes.byref(channels), ctypes.byref(rate)),
                          'sb_pcm_info')
            if check is not None:
                check(frames.value)

            def load(padding, total):
                raw = ctypes.c_void_p()
                with nvtx_range('sushi_b200: sb_pcm_load'):
                    _native.check(lib.sb_pcm_load(h, sample_rate, padding, total, ctypes.byref(raw)), 'sb_pcm_load')
                return raw
            self._load_gpu_with(load, frames.value, rate.value, sample_rate, sample_type, device)
        finally:
            lib.sb_pcm_destroy(h)

    def _load_gpu(self, pcm, frames, channels, sample_width, framerate, sample_rate, sample_type, device):
        """wav.py:108-156 on the GPU: geometry here (same scalar code as the reference), arithmetic
        in sb_load_pcm / sb_normalise; .data is then mirrored back for get_substream views.  `frames` is the
        header's frame count, which sizes the stream; `pcm` is every byte the chunk loop reads, which may be more or
        fewer frames (a partial frame at its end is dropped, as readframes drops it)."""
        if sample_width not in (2, 3):
            raise SushiError('Unsupported sample width: {0}'.format(sample_width))
        decoded = len(pcm) // (channels * sample_width)
        buf = np.frombuffer(pcm, dtype=np.uint8, count=decoded * channels * sample_width)

        def load(padding, total):
            raw = ctypes.c_void_p()
            with nvtx_range('sushi_b200: sb_load_pcm'):
                _native.check(lib.sb_load_pcm(buf.ctypes.data_as(ctypes.c_void_p), decoded, channels, sample_width,
                                              framerate, sample_rate, padding, total, ctypes.byref(raw)), 'sb_load_pcm')
            return raw
        lib = _native.lib(device)
        self._load_gpu_with(load, frames, framerate, sample_rate, sample_type, device)

    def _load_gpu_with(self, load, frames, framerate, sample_rate, sample_type, device):
        """The geometry of wav.py:113-120 for `frames` frames at `framerate`, then load(padding, total) -> the raw
        float32 stream (sb_load_pcm or sb_pcm_load), normalised by sb_normalise and mirrored back."""
        total_seconds = frames / float(framerate)
        self.sample_count = math.ceil(total_seconds * sample_rate)
        self.sample_rate = sample_rate
        self.sample_type = sample_type
        self.padding_size = 10 * framerate
        total = int(self.PADDING_SECONDS * 2 * framerate + self.sample_count)
        lib = _native.lib(device)
        raw = load(self.padding_size, total)
        h = ctypes.c_void_p()
        lo, hi = ctypes.c_float(), ctypes.c_float()
        try:
            with nvtx_range('sushi_b200: sb_normalise'):
                _native.check(lib.sb_normalise(raw, _DTYPES[sample_type][1], ctypes.byref(h), ctypes.byref(lo),
                                               ctypes.byref(hi)), 'sb_normalise')
        finally:
            lib.sb_stream_destroy(raw)
        self.min_value, self.max_value = lo.value, hi.value
        self._handle = h
        self._lib = lib
        self.data = np.empty((1, total), _DTYPES[sample_type][0])
        _native.check(lib.sb_stream_read(h, 0, total, self.data.ctypes.data_as(ctypes.c_void_p)), 'sb_stream_read')
        self._base = self.data.__array_interface__['data'][0]
        _live_streams.add(self)

    # -- construction -----------------------------------------------------------------
    def _load(self, stream, sample_rate, sample_type):
        framerate = stream.framerate
        total_seconds = stream.frames_count / float(framerate)
        downsample_rate = sample_rate / float(framerate)
        self.sample_count = math.ceil(total_seconds * sample_rate)
        self.sample_rate = sample_rate
        self.sample_type = sample_type
        self.padding_size = 10 * framerate          # file-rate samples, as in wav.py:120
        total = int(self.PADDING_SECONDS * 2 * framerate + self.sample_count)
        # np.empty in the reference; fresh pages read as zero, so do ours
        data = np.zeros((1, total), np.float32)
        chunk_frames = int(self.READ_CHUNK_SIZE * framerate)
        pos = self.padding_size
        seconds_read = 0
        maps = {}
        while seconds_read < total_seconds:
            mono = stream.readframes(chunk_frames)
            new_length = int(py2_round(len(mono) * downsample_rate))
            if not new_length:
                # a last chunk too short for one output sample: the reference's cv2.resize raises here; this
                # loader, like the GPU one, takes no sample from it (DESIGN.md section 2)
                mono = mono[:0]
            elif downsample_rate != 1:
                key = (len(mono), new_length)
                if key not in maps:
                    maps[key] = nearest_index_map(*key)
                mono = mono[maps[key]]
            data[0, pos:pos + new_length] = mono
            pos += new_length
            seconds_read += self.READ_CHUNK_SIZE
        data[0, 0:self.padding_size] = data[0, self.padding_size]
        data[0, -self.padding_size:] = data[0, -self.padding_size - 1]
        self.data, self.min_value, self.max_value = normalise_host(data, sample_type)

    @classmethod
    def from_pcm(cls, pcm, framerate, sample_rate=12000, sample_type='uint8', channels=1, device=None, loader='gpu'):
        """Build a stream from an in-memory int16 array (frames x channels, interleaved) --
        the same pipeline as a file load without the RIFF walk (synthetic benches/tests)."""
        pcm = np.ascontiguousarray(pcm, dtype='<i2')
        if sample_type not in _DTYPES:
            raise SushiError('Unknown sample type of WAV stream, must be uint8 or float32')
        self = object.__new__(cls)
        self._handle = None
        raw = pcm.reshape(-1).view(np.uint8).tobytes()
        if loader == 'gpu':
            self._load_gpu(raw, pcm.size // channels, channels, 2, framerate, sample_rate, sample_type, device)
        else:
            self._load(DownmixedWavFile.from_bytes(raw, channels, framerate, 2), sample_rate, sample_type)
            self._upload(device)
        return self

    @classmethod
    def from_array(cls, data, sample_rate, padding_size, sample_count, device=None):
        """Wrap an already-normalised (1,N) uint8/float32 array (what WavStream.data holds)."""
        data = np.ascontiguousarray(data)
        if data.ndim != 2 or data.shape[0] != 1 or data.dtype not in (np.uint8, np.float32):
            raise SushiError('from_array expects a (1,N) uint8 or float32 array')
        self = object.__new__(cls)
        self._handle = None
        self.data = data
        self.sample_rate = sample_rate
        self.sample_type = 'uint8' if data.dtype == np.uint8 else 'float32'
        self.padding_size = int(padding_size)
        self.sample_count = sample_count
        self.min_value = self.max_value = None
        self._upload(device)
        return self

    @classmethod
    def from_device(cls, dev_ptr, n, sample_type, sample_rate, padding_size, sample_count, host_mirror=None, device=None):
        """Wrap n normalised samples that already sit in GPU memory (e.g. an NCCL broadcast buffer);
        they are copied device-to-device into a library-owned stream.  `host_mirror` optionally
        provides .data for get_substream views; without it only the planned/batched calls work."""
        self = object.__new__(cls)
        self._handle = None
        self.data = host_mirror
        self._total = int(n)
        self.sample_rate = sample_rate
        self.sample_type = sample_type
        self.padding_size = int(padding_size)
        self.sample_count = sample_count
        self.min_value = self.max_value = None
        lib = _native.lib(device)
        h = ctypes.c_void_p()
        _native.check(lib.sb_stream_create_device(ctypes.c_void_p(int(dev_ptr)), int(n), _DTYPES[sample_type][1],
                                                  ctypes.byref(h)), 'sb_stream_create_device')
        self._handle = h
        self._lib = lib
        self._base = host_mirror.__array_interface__['data'][0] if host_mirror is not None else 0
        if host_mirror is not None:
            _live_streams.add(self)
        return self

    @property
    def device_ptr(self):
        return self._lib.sb_stream_device_ptr(self._handle)

    def find_planned_device(self, src_stream, toff, tlen, lag0, nlags, d_diff_ptr, d_idx_ptr):
        """Enqueue a planned batch; results (float32[count], int64[count]) land in device memory."""
        arrs = [np.ascontiguousarray(x, dtype=np.int64) for x in (toff, tlen, lag0, nlags)]
        _native.check(self._lib.sb_find_batch_device(
            self._handle, src_stream._handle, len(arrs[0]),
            *[x.ctypes.data_as(_native.c_i64p) for x in arrs],
            ctypes.c_void_p(int(d_diff_ptr)), ctypes.c_void_p(int(d_idx_ptr))), 'sb_find_batch_device')

    def _upload(self, device):
        lib = _native.lib(device)
        h = ctypes.c_void_p()
        _native.check(lib.sb_stream_create(self.data.ctypes.data_as(ctypes.c_void_p), self.data.shape[1],
                                           _DTYPES[self.sample_type][1], ctypes.byref(h)), 'sb_stream_create')
        self._handle = h
        self._lib = lib
        self._base = self.data.__array_interface__['data'][0]
        _live_streams.add(self)

    def close(self):
        if getattr(self, '_handle', None) is not None and self._handle:
            self._lib.sb_stream_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- the reference's surface (duration_seconds, _get_sample_for_time: StreamGeometry) ----
    def get_substream(self, start, end):
        start_off = self._get_sample_for_time(start)
        end_off = self._get_sample_for_time(end)
        return self.data[:, start_off:end_off]

    def _window(self, pattern_len, window_center, window_size):
        """Integer search span of one find_substream call: (start_time, first sample, sample count)."""
        start_time = clip(window_center - window_size, -self.PADDING_SECONDS, self.duration_seconds)
        end_time = clip(window_center + window_size, 0, self.duration_seconds + self.PADDING_SECONDS)
        start_sample = self._get_sample_for_time(start_time)
        end_sample = self._get_sample_for_time(end_time) + pattern_len
        lo, hi, _ = slice(start_sample, end_sample).indices(self.total_samples)   # numpy slice rules (wav.py:184)
        return start_time, lo, max(hi - lo, 0)

    def _locate(self, pattern):
        """(stream, offset) if `pattern` is a contiguous view into a live stream's .data, else None."""
        if not isinstance(pattern, np.ndarray) or pattern.ndim != 2 or pattern.shape[0] != 1:
            return None
        if pattern.shape[1] > 1 and pattern.strides[1] != pattern.itemsize:
            return None
        addr = pattern.__array_interface__['data'][0]
        for s in _live_streams:
            if s._handle and s.data.dtype == pattern.dtype:
                off = addr - s._base
                if 0 <= off and off + pattern.nbytes <= s.data.nbytes and off % s.data.itemsize == 0:
                    return s, off // s.data.itemsize
        return None

    def find_substream(self, pattern, window_center, window_size):
        n = len(pattern[0])
        if pattern.dtype != self.data.dtype:
            raise SushiError('pattern dtype {0} does not match stream dtype {1}'.format(pattern.dtype, self.data.dtype))
        start_time, lo, span = self._window(n, window_center, window_size)
        if n < 1 or span < 1:
            raise SushiError('find_substream: empty pattern or empty search span')
        diff = ctypes.c_float()
        idx = ctypes.c_int64()
        where = self._locate(pattern)
        if span >= n:
            cached = self._from_cache(where, n, lo, span - n + 1)
            if cached is not None:
                return np.float32(cached[0]), start_time + (cached[1] / float(self.sample_rate))
            if where is not None:
                src, off = where
                a = (ctypes.c_int64 * 4)(off, n, lo, span - n + 1)
                _native.check(self._lib.sb_find_batch(
                    self._handle, src._handle, 1,
                    ctypes.cast(ctypes.byref(a, 0), _native.c_i64p), ctypes.cast(ctypes.byref(a, 8), _native.c_i64p),
                    ctypes.cast(ctypes.byref(a, 16), _native.c_i64p), ctypes.cast(ctypes.byref(a, 24), _native.c_i64p),
                    ctypes.byref(diff), ctypes.byref(idx)), 'sb_find_batch')
            else:
                pat = np.ascontiguousarray(pattern[0])
                _native.check(self._lib.sb_find(self._handle, pat.ctypes.data_as(ctypes.c_void_p), n, lo,
                                                span - n + 1, ctypes.byref(diff), ctypes.byref(idx)), 'sb_find')
        else:
            # search span shorter than the pattern: cv2.matchTemplate silently swaps image and
            # template (survey appendix A); mirror that instead of failing
            if where is None:
                tmp = WavStream.from_array(np.ascontiguousarray(pattern), self.sample_rate, 0, n)
                src, off = tmp, 0
            else:
                src, off = where
            a = (ctypes.c_int64 * 4)(lo, span, off, n - span + 1)
            _native.check(self._lib.sb_find_batch(
                src._handle, self._handle, 1,
                ctypes.cast(ctypes.byref(a, 0), _native.c_i64p), ctypes.cast(ctypes.byref(a, 8), _native.c_i64p),
                ctypes.cast(ctypes.byref(a, 16), _native.c_i64p), ctypes.cast(ctypes.byref(a, 24), _native.c_i64p),
                ctypes.byref(diff), ctypes.byref(idx)), 'sb_find_batch')
        return np.float32(diff.value), start_time + (idx.value / float(self.sample_rate))

    def find_substream_many(self, queries):
        """[(pattern, center, window), ...] -> [(np.float32, float), ...] in ONE launch when every
        pattern is a view into a resident stream of the same source (the whole/left/right probes of
        the shift solver, sushi.py:450-452); otherwise falls back to one call each."""
        plan = []
        src = None
        for pattern, center, window in queries:
            where = self._locate(pattern) if pattern.dtype == self.data.dtype else None
            n = len(pattern[0])
            start_time, lo, span = self._window(n, center, window)
            if where is None or (src is not None and where[0] is not src) or n < 1 or span < n:
                return [self.find_substream(*q) for q in queries]
            src = where[0]
            plan.append((where[1], n, lo, span - n + 1, start_time))
        toff, tlen, lag0, nlags, t0 = zip(*plan)
        diff, idx = self.find_planned(src, toff, tlen, lag0, nlags)
        rate = float(self.sample_rate)
        return [(np.float32(diff[q]), t0[q] + (int(idx[q]) / rate)) for q in range(len(plan))]

    # -- batched surface (what the sharded benchmark and the batched shift solver use) ------
    def find_substream_batch(self, src_stream, starts, ends, centers, windows):
        """Batched find_substream: returns (diffs float32[count], times float64[count])."""
        with nvtx_range('sushi_b200: find_substream_batch'):
            toff, tlen, lag0, nlags, t0 = self.plan_queries(src_stream, starts, ends, centers, windows)
            diff, idx = self.find_planned(src_stream, toff, tlen, lag0, nlags)
        return diff, t0 + idx / float(self.sample_rate)

    def find_planned(self, src_stream, toff, tlen, lag0, nlags):
        count = len(toff)
        diff = np.empty(count, np.float32)
        idx = np.empty(count, np.int64)
        arrs = [np.ascontiguousarray(x, dtype=np.int64) for x in (toff, tlen, lag0, nlags)]
        _native.check(self._lib.sb_find_batch(
            self._handle, src_stream._handle, count,
            *[x.ctypes.data_as(_native.c_i64p) for x in arrs],
            diff.ctypes.data_as(_native.c_f32p), idx.ctypes.data_as(_native.c_i64p)), 'sb_find_batch')
        return diff, idx

    def match_curves(self, src_stream, toff, tlen, lag0, nlags):
        """Whole curves of several queries from one launch: list of float32 arrays."""
        arrs = [np.ascontiguousarray(x, dtype=np.int64) for x in (toff, tlen, lag0, nlags)]
        out = np.empty(int(arrs[3].sum()), np.float32)
        _native.check(self._lib.sb_match_curves(self._handle, src_stream._handle, len(arrs[0]),
                                                *[x.ctypes.data_as(_native.c_i64p) for x in arrs],
                                                out.ctypes.data_as(_native.c_f32p)), 'sb_match_curves')
        cuts = np.cumsum(arrs[3])[:-1]
        return np.split(out, cuts)

    # -- speculation for the sequential shift solver ------------------------------------------
    SPECULATE_GROUPS = 48        # groups precomputed per launch
    SPECULATE_MARGIN = 0.35      # seconds of slack either side of the predicted search span

    def speculate_fast_path(self, src_stream, groups, idx, anchor, window):
        """Hint from calculate_shifts: groups[idx:] are about to be searched one by one around
        start + anchor with +-window (the fast path, sushi.py:431-432).  Precompute, in ONE launch, the
        curves of the next groups over a slightly wider span; find_substream then answers from them.
        A curve value depends only on (template, absolute position), so a cached curve answers any
        contained range with exactly the value and first-index argmin a live call returns (every engine
        computes a value the same way whatever the batch)."""
        plan = self._speculation_plan(src_stream, groups, idx, anchor, window)
        if plan is not None:
            self._fill_curve_cache(src_stream, plan, self.match_curves(src_stream, *plan))

    def _speculation_plan(self, src_stream, groups, idx, anchor, window):
        """The queries speculate_fast_path would precompute, (toff, tlen, lag0, nlags), or None when the cache already
        holds the group's curve or no group fits its search span."""
        cache = self.__dict__.setdefault('_curve_cache', {})
        # keys are the CLAMPED template ranges, the same integers find_substream derives from a view.  This runs once
        # per search group: the common case (the group's curve is there) must cost a few scalar operations, not arrays
        # over the next 48 groups
        if cache:
            total, pad, rate = src_stream.total_samples, src_stream.padding_size, src_stream.sample_rate
            lo = int(rate * float(groups[idx][0].start)) + pad          # trunc toward zero, like plan_queries
            hi = int(rate * float(groups[idx][-1].end)) + pad
            lo = max(lo + total, 0) if lo < 0 else min(lo, total)
            hi = max(hi + total, 0) if hi < 0 else min(hi, total)
            if (lo, lo + max(hi - lo, 0)) in cache:
                return None
        batch = groups[idx:idx + self.SPECULATE_GROUPS]
        starts = np.array([g[0].start for g in batch], np.float64)
        ends = np.array([g[-1].end for g in batch], np.float64)
        windows = np.full(len(batch), window + self.SPECULATE_MARGIN)
        cache.clear()                                        # predictions made for an older anchor
        try:
            toff, tlen, lag0, nlags, _ = self.plan_queries(src_stream, starts, ends, starts + anchor, windows)
        except SushiError:
            # some group does not fit its search span (end of the stream): keep the ones that do
            keep = []
            for q in range(len(batch)):
                try:
                    self.plan_queries(src_stream, starts[q:q + 1], ends[q:q + 1], starts[q:q + 1] + anchor, windows[q:q + 1])
                    keep.append(q)
                except SushiError:
                    pass
            if not keep:
                return None
            toff, tlen, lag0, nlags, _ = self.plan_queries(src_stream, starts[keep], ends[keep], starts[keep] + anchor,
                                                           windows[keep])
        return toff, tlen, lag0, nlags

    def _fill_curve_cache(self, src_stream, plan, curves):
        toff, tlen, lag0, _ = plan
        cache = self.__dict__.setdefault('_curve_cache', {})
        for q in range(len(toff)):
            cache[(int(toff[q]), int(toff[q] + tlen[q]))] = (src_stream, int(lag0[q]), curves[q])

    def _from_cache(self, where, n, lo, nlags):
        cache = self.__dict__.get('_curve_cache')
        if not cache or where is None:
            return None
        hit = cache.get((where[1], where[1] + n))
        if hit is None or hit[0] is not where[0]:
            return None
        _, c_lo, curve = hit
        a = lo - c_lo
        if a < 0 or a + nlags > len(curve):
            return None
        part = curve[a:a + nlags]
        i = int(part.argmin())                               # first of equal minima, like the kernel
        return part[i], i

    def match_curve(self, src_stream, toff, tlen, lag0, nlags):
        """Whole TM_SQDIFF_NORMED curve of one query (parity tests / debugging)."""
        out = np.empty(int(nlags), np.float32)
        _native.check(self._lib.sb_match_curve(self._handle, src_stream._handle, int(toff), int(tlen), int(lag0),
                                               int(nlags), out.ctypes.data_as(_native.c_f32p)), 'sb_match_curve')
        return out


# -- many streams at once (sb_find_multi / sb_match_curves_multi) ---------------------------------
def _multi_arrays(pairs):
    """[(image_stream, tmpl_stream), ...] -> (stream table, image slots, template slots) of one multi-stream call."""
    slot, handles = {}, []
    islot = np.empty(len(pairs), np.int32)
    tslot = np.empty(len(pairs), np.int32)
    for q, (img, tmpl) in enumerate(pairs):
        for s, out in ((img, islot), (tmpl, tslot)):
            if id(s) not in slot:
                slot[id(s)] = len(handles)
                handles.append(s._handle)
            out[q] = slot[id(s)]
    table = (ctypes.c_void_p * len(handles))(*[h.value for h in handles])
    return table, len(handles), islot, tslot


def _by_dtype(items, key):
    groups = {}
    for i, it in enumerate(items):
        groups.setdefault(key(it), []).append(i)
    return groups.values()


def find_substreams(requests):
    """[(dst_stream, pattern, window_center, window_size), ...] -> [(np.float32, float), ...]: for every request exactly
    what dst_stream.find_substream(pattern, window_center, window_size) returns.  Requests whose pattern is a view of a
    live stream go out together in ONE sb_find_multi per sample type, whatever their streams (a curve cached by
    speculate_fast_path answers on the host, as in find_substream); anything else -- detached copies, a search span
    shorter than the pattern -- goes through dst_stream.find_substream."""
    out = [None] * len(requests)
    live = []
    for r, (dst, pattern, center, window) in enumerate(requests):
        where = dst._locate(pattern) if pattern.dtype == dst.data.dtype else None
        n = len(pattern[0])
        start_time, lo, span = dst._window(n, center, window)
        if where is None or n < 1 or span < n:
            out[r] = dst.find_substream(pattern, center, window)
            continue
        cached = dst._from_cache(where, n, lo, span - n + 1)
        if cached is not None:
            out[r] = (np.float32(cached[0]), start_time + (cached[1] / float(dst.sample_rate)))
            continue
        live.append((r, dst, where[0], where[1], n, lo, span - n + 1, start_time))
    for sel in _by_dtype(live, lambda x: x[1].data.dtype):
        part = [live[i] for i in sel]
        table, n_streams, islot, tslot = _multi_arrays([(x[1], x[2]) for x in part])
        arrs = [np.ascontiguousarray([x[k] for x in part], dtype=np.int64) for k in (3, 4, 5, 6)]
        diff = np.empty(len(part), np.float32)
        idx = np.empty(len(part), np.int64)
        lib = part[0][1]._lib
        _native.check(lib.sb_find_multi(table, n_streams, len(part), islot.ctypes.data_as(_native.c_i32p),
                                        tslot.ctypes.data_as(_native.c_i32p), *[a.ctypes.data_as(_native.c_i64p) for a in arrs],
                                        diff.ctypes.data_as(_native.c_f32p), idx.ctypes.data_as(_native.c_i64p)), 'sb_find_multi')
        for q, x in enumerate(part):
            out[x[0]] = (np.float32(diff[q]), x[7] + (int(idx[q]) / float(x[1].sample_rate)))
    return out


def match_curves_multi(requests):
    """[(dst_stream, src_stream, toff, tlen, lag0, nlags), ...] with descriptor arrays per request -> per request the list
    of curves dst_stream.match_curves(src_stream, toff, tlen, lag0, nlags) returns; one sb_match_curves_multi per
    sample type."""
    out = [None] * len(requests)
    for sel in _by_dtype(requests, lambda r: r[0].data.dtype):
        pairs, cols, counts = [], [[], [], [], []], []
        for i in sel:
            dst, src, toff, tlen, lag0, nlags = requests[i]
            counts.append(len(toff))
            pairs += [(dst, src)] * len(toff)
            for k, a in enumerate((toff, tlen, lag0, nlags)):
                cols[k] += [int(v) for v in a]
        if not pairs:
            for i in sel:
                out[i] = []
            continue
        table, n_streams, islot, tslot = _multi_arrays(pairs)
        arrs = [np.ascontiguousarray(c, dtype=np.int64) for c in cols]
        curves = np.empty(int(arrs[3].sum()), np.float32)
        lib = requests[sel[0]][0]._lib
        _native.check(lib.sb_match_curves_multi(table, n_streams, len(pairs), islot.ctypes.data_as(_native.c_i32p),
                                                tslot.ctypes.data_as(_native.c_i32p), *[a.ctypes.data_as(_native.c_i64p) for a in arrs],
                                                curves.ctypes.data_as(_native.c_f32p)), 'sb_match_curves_multi')
        pieces = np.split(curves, np.cumsum(arrs[3])[:-1])
        at = 0
        for i, cnt in zip(sel, counts):
            out[i] = pieces[at:at + cnt]
            at += cnt
    return out


def speculate_fast_path_many(requests):
    """[(dst_stream, src_stream, groups, idx, anchor, window), ...]: speculate_fast_path for every request, with the
    curves of all of them from ONE sb_match_curves_multi.  Each destination's cache is filled, keyed exactly like
    speculate_fast_path's; two requests on one destination evict each other's entries (later live calls are slower,
    never different)."""
    todo = []
    for dst, src, groups, idx, anchor, window in requests:
        plan = dst._speculation_plan(src, groups, idx, anchor, window)
        if plan is not None:
            todo.append((dst, src, plan))
    if not todo:
        return
    curves = match_curves_multi([(dst, src) + tuple(plan) for dst, src, plan in todo])
    for (dst, src, plan), c in zip(todo, curves):
        dst._fill_curve_cache(src, plan, c)
