"""The reference's run() after demuxing (sushi.py:653-726) as a function: load both streams, prepare
the search groups, solve the shifts, post-process them with the grouping heuristics, correct them
against video keyframes when keyframe times are given, move the events.  Demuxing, making keyframes
or timecodes from video and plotting are outside this path (DESIGN.md section 0); the command line
on top of it is sushi_b200.cli.
"""
import logging

from .common import format_time
from .grouping import (average_shifts, detect_groups, fix_near_borders, groups_from_chapters,
                       prepare_search_groups, smooth_events, snap_groups_to_keyframes, split_broken_groups)
from .script import load_script
from .shifts import calculate_shifts, calculate_shifts_many
from .wavstream import WavStream


def shift_events(events, src_stream, dst_stream, chapter_times=(), window=10, max_window=30, rewind_thresh=5,
                 grouping=True, smooth_radius=3, max_ts_duration=1001.0 / 24000.0 * 10,
                 max_ts_distance=1001.0 / 24000.0 * 10, keyframes=None, max_kf_distance=2, kf_mode='all'):
    """Defaults are the reference's command-line defaults (sushi.py:742-765).  `keyframes` is a
    timing.KeyframeTimes (timing.load_keyframe_times); when given, the shifts are snapped to keyframes
    as `--src/--dst-keyframes` do, and every linked event is resolved first.  Events end up with their
    final .shift/.diff (and keyframe corrections); returns the list of groups the shifts were averaged
    over (empty without grouping)."""
    chapter_times = list(chapter_times)
    search_groups = prepare_search_groups(events, src_stream.duration_seconds, chapter_times,
                                          max_ts_duration, max_ts_distance)
    calculate_shifts(src_stream, dst_stream, search_groups, window, max_window, rewind_thresh if grouping else 0)
    return _postprocess(events, chapter_times, grouping, smooth_radius, keyframes, max_kf_distance, kf_mode,
                        max_ts_duration, max_ts_distance)


def shift_events_many(jobs, window=10, max_window=30, rewind_thresh=5, grouping=True, smooth_radius=3,
                      max_ts_duration=1001.0 / 24000.0 * 10, max_ts_distance=1001.0 / 24000.0 * 10,
                      keyframes=None, max_kf_distance=2, kf_mode='all'):
    """shift_events over many jobs [(events, src_stream, dst_stream[, chapter_times[, keyframes]]), ...]: the search
    groups of every job are solved together by calculate_shifts_many (one multi-stream launch per round for all jobs),
    the heuristics before and after run per job.  A job without its own keyframe times uses `keyframes`.  Every event
    ends up with what shift_events gives it; returns the per-job groups."""
    prepared = []
    for job in jobs:
        events, src, dst = job[:3]
        chapter_times = list(job[3]) if len(job) > 3 else []
        job_keyframes = job[4] if len(job) > 4 else keyframes
        prepared.append((events, src, dst, chapter_times, job_keyframes,
                         prepare_search_groups(events, src.duration_seconds, chapter_times, max_ts_duration, max_ts_distance)))
    calculate_shifts_many([(src, dst, groups) for _, src, dst, _, _, groups in prepared], window, max_window,
                          rewind_thresh if grouping else 0)
    return [_postprocess(events, chapter_times, grouping, smooth_radius, job_keyframes, max_kf_distance, kf_mode,
                         max_ts_duration, max_ts_distance)
            for events, _, _, chapter_times, job_keyframes, _ in prepared]


def _postprocess(events, chapter_times, grouping, smooth_radius, keyframes, max_kf_distance, kf_mode,
                 max_ts_duration, max_ts_distance):
    def snap(evs):
        snap_groups_to_keyframes(evs, chapter_times, max_ts_duration, max_ts_distance, keyframes.src_keytimes,
                                 keyframes.dst_keytimes, keyframes.src_timecodes, keyframes.dst_timecodes,
                                 max_kf_distance, kf_mode)

    if not grouping:
        fix_near_borders(events)
        if keyframes is not None:
            _resolve_links(events)
            snap(events)
        return []
    if chapter_times:
        groups = groups_from_chapters(events, chapter_times)
        for g in groups:
            fix_near_borders(g)
            smooth_events([e for e in g if not e.linked], smooth_radius)
        groups = split_broken_groups(groups)
    else:
        fix_near_borders(events)
        smooth_events([e for e in events if not e.linked], smooth_radius)
        groups = detect_groups(events)
    for g in groups:
        first, last = g[0].shift, g[-1].shift
        avg = average_shifts(g)
        logging.info('Group (start: {0}, end: {1}, lines: {2}), shifts (start: {3}, end: {4}, average: {5})'.format(
            format_time(g[0].start), format_time(g[-1].end), len(g), first, last, avg))
    if keyframes is not None:
        _resolve_links(events)
        for g in groups:
            snap(g)
    return groups


def _resolve_links(events):
    # in list order, as sushi.py:707-708: a link to a later linked event still reads through its chain
    for e in events:
        if e.linked:
            e.resolve_link()


def shift_script(src_audio, dst_audio, script_path, output_path, sample_rate=12000, sample_type='uint8',
                 chapter_times=(), src_track=None, dst_track=None, ffmpeg_audio=False, **options):
    """src/dst audio (whatever WavStream takes: a file of a format in inputs.READERS, or an opened container reader) +
    ASS/SRT script in, shifted script out (the audio-in/script-out core of the CLI).
    src_track / dst_track are the audio stream ids of container inputs (None: the reference's default rule).
    ffmpeg_audio loads inputs other than WAV files as the reference's ffmpeg call writes them (WavStream).
    `options` are shift_events' keyword arguments, keyframes included."""
    script = load_script(script_path)
    script.sort_by_time()
    src = WavStream(src_audio, sample_rate=sample_rate, sample_type=sample_type, track=src_track,
                    ffmpeg_audio=ffmpeg_audio)
    dst = WavStream(dst_audio, sample_rate=sample_rate, sample_type=sample_type, track=dst_track,
                    ffmpeg_audio=ffmpeg_audio)
    groups = shift_events(script.events, src, dst, chapter_times=chapter_times, **options)
    for e in script.events:
        e.apply_shift()
    script.save_to_file(output_path)
    return script, groups


def shift_scripts(jobs, sample_rate=12000, sample_type='uint8', **options):
    """shift_script over many jobs [(src_audio, dst_audio, script_path, output_path[, chapter_times[, keyframes]]),
    ...]: every stream is loaded, the shifts of all jobs are solved together (shift_events_many) and every script is
    written -- the same files as one shift_script call per job.  Returns [(script, groups), ...]."""
    scripts, streams = [], []
    for job in jobs:
        src_audio, dst_audio, script_path = job[:3]
        script = load_script(script_path)
        script.sort_by_time()
        scripts.append(script)
        streams.append((WavStream(src_audio, sample_rate=sample_rate, sample_type=sample_type),
                        WavStream(dst_audio, sample_rate=sample_rate, sample_type=sample_type)))
    groups = shift_events_many([(script.events, src, dst, job[4] if len(job) > 4 else ()) + tuple(job[5:6])
                                for script, (src, dst), job in zip(scripts, streams, jobs)], **options)
    for script, job in zip(scripts, jobs):
        for e in script.events:
            e.apply_shift()
        script.save_to_file(job[3])
    return list(zip(scripts, groups))
