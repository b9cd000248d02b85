"""Video-side inputs of keyframe snapping: frame timecodes, keyframe lists and chapter files.
Behavioural mirror of the reference's demux.Timecodes (demux.py:135-224), keyframes.py and the
parsers of chapters.py:5-32.  Everything here is host-side text parsing; making keyframes or
timecodes from a video (SCXvid, mkvextract, ffmpeg) is not part of this project.
"""
import bisect
import collections
import re

from .common import SushiError


def read_all_text(path):
    with open(path) as f:
        return f.read()


class Timecodes(object):
    """Per-frame start times of a video, from a v1 or v2 timecodes file (demux.py:135-207)."""

    def __init__(self, times, default_fps):
        self.times = times
        self.default_frame_duration = 1.0 / default_fps if default_fps else None

    def get_frame_time(self, number):
        try:
            return self.times[number]
        except IndexError:
            if not self.default_frame_duration:
                # v2 lists have no default rate: every frame past the end starts at the last time
                return self.get_frame_time(len(self.times) - 1)
            if self.times:
                return self.times[-1] + (self.default_frame_duration) * (number - len(self.times) + 1)
            return number * self.default_frame_duration

    def get_frame_size(self, timestamp):
        try:
            number = bisect.bisect_left(self.times, timestamp)
        except Exception:
            return self.default_frame_duration
        c = self.get_frame_time(number)
        if number == len(self.times):
            return c - self.get_frame_time(number - 1)
        return self.get_frame_time(number + 1) - c

    @classmethod
    def _convert_v1_to_v2(cls, default_fps, overrides):
        # (start frame, end frame, fps) ranges over a default rate -> frame start times
        overrides = [(int(x[0]), int(x[1]), float(x[2])) for x in overrides]
        if not overrides:
            return []
        fps = [default_fps] * (overrides[-1][1] + 1)      # ends at the LAST override, not the largest end
        for start, end, rate in overrides:
            fps[start:end + 1] = [rate] * (end - start + 1)
        v2 = [0]
        for d in (1.0 / f for f in fps):
            v2.append(v2[-1] + d)
        return v2

    @classmethod
    def parse(cls, text):
        lines = text.splitlines()
        if not lines:
            # the reference returns [] here (demux.py:191-192) and fails later on its first use
            raise SushiError('Timecodes file is empty')
        first = lines[0].lower().lstrip()
        if first.startswith('# timecode format v2') or first.startswith('# timestamp format v2'):
            return Timecodes([float(x) / 1000.0 for x in lines[1:]], None)
        if first.startswith('# timecode format v1'):
            default = float(lines[1].lower().replace('assume ', ''))
            overrides = (x.split(',') for x in lines[2:])
            return Timecodes(cls._convert_v1_to_v2(default, overrides), default)
        raise SushiError('This timecodes format is not supported')

    @classmethod
    def from_file(cls, path):
        return cls.parse(read_all_text(path))

    @classmethod
    def cfr(cls, fps):
        return CfrTimecodes(fps)


class CfrTimecodes(object):
    """Constant frame rate: what `--src-fps/--dst-fps` stand for (demux.py:209-224)."""

    def __init__(self, fps):
        self.frame_duration = 1.0 / fps

    def get_frame_time(self, number):
        return number * self.frame_duration

    def get_frame_size(self, timestamp):
        return self.frame_duration


def parse_scxvid_keyframes(text):
    """Frame numbers of the 'i' lines of an XviD 2-pass stat file; frame 0 is the 4th line."""
    return [i - 3 for i, line in enumerate(text.splitlines()) if line and line[0] == 'i']


def parse_keyframes(path):
    text = read_all_text(path)
    if '# XviD 2pass stat file' not in text:
        raise SushiError('Unsupported keyframes type')
    frames = parse_scxvid_keyframes(text)
    if 0 not in frames:
        frames.insert(0, 0)
    return frames


def _parse_chapter_times(times):
    result = []
    for t in times:
        hours, minutes, seconds = map(float, t.split(':'))
        result.append(hours * 3600 + minutes * 60 + seconds)
    result.sort()
    if result[0] != 0:        # a file without chapters raises IndexError here, as in the reference (chapters.py:12)
        result.insert(0, 0)
    return result


def parse_xml_start_times(text):
    """Chapter start times of a Matroska XML chapters file, sorted, with 0 first."""
    return _parse_chapter_times(re.findall(r'<ChapterTimeStart>(\d+:\d+:\d+\.\d+)</ChapterTimeStart>', text))


def get_xml_start_times(path):
    return parse_xml_start_times(read_all_text(path))


def parse_ogm_start_times(text):
    """Chapter start times of an OGM (CHAPTERnn=hh:mm:ss.sss) chapters file, sorted, with 0 first."""
    return _parse_chapter_times(re.findall(r'CHAPTER\d+=(\d+:\d+:\d+\.\d+)', text, flags=re.IGNORECASE))


def get_ogm_start_times(path):
    return parse_ogm_start_times(read_all_text(path))


KeyframeTimes = collections.namedtuple('KeyframeTimes', ['src_keytimes', 'dst_keytimes', 'src_timecodes', 'dst_timecodes'])


def load_keyframe_times(src_keyframes, dst_keyframes, src_fps=None, dst_fps=None, src_timecodes=None, dst_timecodes=None):
    """Keyframe times of both videos from their keyframe files, each on its own timecodes: a constant
    rate when its fps is given, otherwise its timecodes file (sushi.py:653-658).  The result is what
    the `keyframes=` argument of shift_events / shift_script takes."""
    src_tc = Timecodes.cfr(src_fps) if src_fps else Timecodes.from_file(src_timecodes)
    src_keytimes = [src_tc.get_frame_time(f) for f in parse_keyframes(src_keyframes)]
    dst_tc = Timecodes.cfr(dst_fps) if dst_fps else Timecodes.from_file(dst_timecodes)
    dst_keytimes = [dst_tc.get_frame_time(f) for f in parse_keyframes(dst_keyframes)]
    return KeyframeTimes(src_keytimes, dst_keytimes, src_tc, dst_tc)
