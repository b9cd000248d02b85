"""Small helpers shared by the host side (mirror of the pieces of the reference's
common.py that the hot path touches: SushiError common.py:4, clip common.py:41-42,
format_time common.py:32-38 -- used only in log lines)."""
import collections
import logging


class SushiError(Exception):
    """User-facing failure; the reference's CLI prints it and exits 2 (sushi.py:841-843)."""


# What every reader's select_audio(track) returns, once each refusal that needs no GPU has passed: the audio WavStream
# loads.  `label` names a codec the GPU decodes ('FLAC', 'TrueHD', 'BD-LPCM', ...) and is None for PCM; `id` is the
# stream id in a container; `path` names the file in messages.  A codec has decode(device) -> the sb_pcm handle of the
# decoded samples (it loads the library, and reads a container track's frames first) and may have check(frames), which
# refuses the decoded frame count; PCM has pcm() -> (bytes, frames, channels, sample width, rate, big-endian).  For the
# --ffmpeg-audio conversion (sushi_b200/swr.py) a reader also tells what FFmpeg's decoder outputs: `fmt` its sample
# format ('S16' or 'S32'; None when the reader cannot tell before decoding), `bits` the source's bit depth, and
# `layout` its channel mask (AV_CH_* bits) by channel count.
Audio = collections.namedtuple('Audio', 'label id path decode pcm check fmt bits layout', defaults=(None,) * 8)


def clip(value, minimum, maximum):
    # reference common.py:41-42 -- note the order: min() first, then max()
    return max(min(value, maximum), minimum)


def py2_round(x):
    """round() as Python 2 does it (half away from zero): the reference is py2 code
    (wav.py:127, common.py:33, subs.py:116)."""
    import math
    return math.floor(x + 0.5) if x >= 0 else -math.floor(-x + 0.5)


def format_time(seconds):
    cs = py2_round(seconds * 100)
    return '{0}:{1:02d}:{2:02d}.{3:02d}'.format(
        int(cs // 360000), int((cs // 6000) % 60), int((cs // 100) % 60), int(cs % 100))


def format_stream(t):
    """One line of a stream candidate list: id, title, what the stream is."""
    return '{0}{1}: {2}'.format(t.id, ' (%s)' % t.title if t.title else '', t.info)


class Container(object):
    """What every container reader (Matroska, MP4, transport and program streams) offers over its stream list
    `self.tracks` (objects with .id, .kind, .title, .info and .default) and the file name `self.path`."""

    def close(self):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def prefetch(self, payload_ids=(), time_ids=()):
        """Nothing to read ahead: the audio is read by WavStream, and there is no script or timestamp to read."""

    @property
    def streams_all(self):
        """Every stream of the file, in its order (the MPEG readers' name for `tracks`)."""
        return self.tracks

    def streams(self, kind):
        return [t for t in self.tracks if t.kind == kind]

    def select(self, kind, idx):
        """The reference's Demuxer._select_stream (demux.py:335-355): kind is 'audio', 'subtitles' or 'video'."""
        return select_stream(self.streams(kind), kind, idx, self.path)


def select_stream(streams, kind, idx, path):
    """The reference's Demuxer._select_stream (demux.py:335-355) over a container's streams of one kind (objects with
    .id, .title, .info and .default): `idx` a stream id, or None for the only stream, else the default one."""
    listing = '\n'.join(format_stream(t) for t in streams)
    if not streams:
        raise SushiError('No {0} streams found in {1}'.format(kind, path))
    if idx is None:
        if len(streams) > 1:
            default = next((t for t in streams if t.default), None)
            if default:
                logging.warning('Using default track {0} in {1} because there are multiple candidates'
                                .format(format_stream(default), path))
                return default
            raise SushiError('More than one {0} stream found in {1}.'
                             'You need to specify the exact one to demux. Here are all candidates:\n'
                             '{2}'.format(kind, path, listing))
        return streams[0]
    try:
        return next(t for t in streams if t.id == idx)
    except StopIteration:
        raise SushiError("Stream with index {0} doesn't exist in {1}.\n"
                         "Here are all that do:\n"
                         "{2}".format(idx, path, listing))
