"""The Sushi command line: `python -m sushi_b200 --src a.mkv --dst b.mkv -o out.ass`.

Flags, defaults and checks are the reference's (sushi.py:528-843).  --src and --dst are files of the formats in
inputs.READERS, taken by their extensions.  For a WAV file the reference starts no subprocess either; any other
format is decoded on the GPU, where the reference would have ffmpeg convert it to a WAV file (DESIGN.md section 2):
no WAV file is ever written.  A Matroska input also gives, as the reference's ffmpeg and
mkvextract calls do, the script, the chapters and the video timestamps (sushi_b200.matroska); those are written to
the reference's temporary paths and removed at the end unless --no-cleanup is given.  Every check runs before the GPU
is touched; the run itself is pipeline.shift_script.
"""
import argparse
import io
import logging
import os
import sys
import time

from . import __version__, swr
from .common import SushiError
from .inputs import READERS
from .pipeline import shift_script
from .script import format_srt_time
from .timing import get_ogm_start_times, get_xml_start_times, load_keyframe_times


def get_extension(path):
    return os.path.splitext(path)[1].lower()


def check_file_exists(path, file_title):
    if path and not os.path.exists(path):
        raise SushiError("{0} file doesn't exist".format(file_title))


def format_full_path(temp_dir, base_path, postfix):
    if temp_dir:
        return os.path.join(temp_dir, os.path.basename(base_path) + postfix)
    return base_path + postfix


def create_directory_if_not_exists(path):
    if path and not os.path.exists(path):
        os.makedirs(path)


def create_arg_parser():
    parser = argparse.ArgumentParser(prog='sushi_b200', description='Sushi - Automatic Subtitle Shifter')

    parser.add_argument('--window', default=10, type=int, metavar='<size>', dest='window',
                        help='Search window size. [%(default)s]')
    parser.add_argument('--max-window', default=30, type=int, metavar='<size>', dest='max_window',
                        help='Maximum search size Sushi is allowed to use when trying to recover from errors. [%(default)s]')
    parser.add_argument('--rewind-thresh', default=5, type=int, metavar='<events>', dest='rewind_thresh',
                        help='Number of consecutive errors Sushi has to encounter to consider results broken '
                             'and retry with larger window. Set to 0 to disable. [%(default)s]')
    parser.add_argument('--no-grouping', action='store_false', dest='grouping',
                        help="Don't events into groups before shifting. Also disables error recovery.")
    parser.add_argument('--max-kf-distance', default=2, type=float, metavar='<frames>', dest='max_kf_distance',
                        help='Maximum keyframe snapping distance. [%(default)s]')
    parser.add_argument('--kf-mode', default='all', choices=['shift', 'snap', 'all'], dest='kf_mode',
                        help='Keyframes-based shift correction/snapping mode. [%(default)s]')
    parser.add_argument('--smooth-radius', default=3, type=int, metavar='<events>', dest='smooth_radius',
                        help='Radius of smoothing median filter. [%(default)s]')

    # 10 frames at 23.976
    parser.add_argument('--max-ts-duration', default=1001.0 / 24000.0 * 10, type=float, metavar='<seconds>',
                        dest='max_ts_duration',
                        help='Maximum duration of a line to be considered typesetting. [%(default).3f]')
    parser.add_argument('--max-ts-distance', default=1001.0 / 24000.0 * 10, type=float, metavar='<seconds>',
                        dest='max_ts_distance',
                        help='Maximum distance between two adjacent typesetting lines to be merged. [%(default).3f]')

    parser.add_argument('--sample-type', default='uint8', choices=['float32', 'uint8'], dest='sample_type',
                        help=argparse.SUPPRESS)
    parser.add_argument('--sample-rate', default=12000, type=int, metavar='<rate>', dest='sample_rate',
                        help='Downsampled audio sample rate. [%(default)s]')
    parser.add_argument('--ffmpeg-audio', action='store_true', dest='ffmpeg_audio',
                        help='Load inputs other than WAV files as the reference\'s ffmpeg call writes them: '
                             'libswresample\'s downmix and resample of 16-bit sources, bit for bit')

    # stream indices select streams of a Matroska input; WAV and FLAC inputs have one of each, so they are ignored
    parser.add_argument('--src-audio', default=None, type=int, metavar='<id>', dest='src_audio_idx',
                        help='Audio stream index of the source video (ignored for WAV and FLAC input)')
    parser.add_argument('--src-script', default=None, type=int, metavar='<id>', dest='src_script_idx',
                        help='Script stream index of the source video (ignored for WAV and FLAC input)')
    parser.add_argument('--dst-audio', default=None, type=int, metavar='<id>', dest='dst_audio_idx',
                        help='Audio stream index of the destination video (ignored for WAV and FLAC input)')

    parser.add_argument('--no-cleanup', action='store_false', dest='cleanup',
                        help="Don't delete demuxed streams")
    parser.add_argument('--temp-dir', default=None, dest='temp_dir', metavar='<string>',
                        help='Specify temporary folder to use when demuxing stream.')
    parser.add_argument('--chapters', default=None, dest='chapters_file', metavar='<filename>',
                        help="XML or OGM chapters to use instead of any found in the source. 'none' to disable.")
    parser.add_argument('--script', default=None, dest='script_file', metavar='<filename>',
                        help='Subtitle file path to use instead of any found in the source')

    parser.add_argument('--dst-keyframes', default=None, dest='dst_keyframes', metavar='<filename>',
                        help='Destination keyframes file')
    parser.add_argument('--src-keyframes', default=None, dest='src_keyframes', metavar='<filename>',
                        help='Source keyframes file')
    parser.add_argument('--dst-fps', default=None, type=float, dest='dst_fps', metavar='<fps>',
                        help='Fps of the destination video. Must be provided if keyframes are used.')
    parser.add_argument('--src-fps', default=None, type=float, dest='src_fps', metavar='<fps>',
                        help='Fps of the source video. Must be provided if keyframes are used.')
    parser.add_argument('--dst-timecodes', default=None, dest='dst_timecodes', metavar='<filename>',
                        help='Timecodes file to use instead of making one from the destination (when possible)')
    parser.add_argument('--src-timecodes', default=None, dest='src_timecodes', metavar='<filename>',
                        help='Timecodes file to use instead of making one from the source (when possible)')

    parser.add_argument('--src', required=True, dest='source', metavar='<filename>',
                        help='Source audio or video (WAV, FLAC, WavPack, TTA, APE, TAK, TrueHD, Matroska, MP4, MPEG-TS, Ogg or AVI)')
    parser.add_argument('--dst', required=True, dest='destination', metavar='<filename>',
                        help='Destination audio or video (WAV, FLAC, WavPack, TTA, APE, TAK, TrueHD, Matroska, MP4, MPEG-TS, Ogg or AVI)')
    parser.add_argument('-o', '--output', default=None, dest='output_script', metavar='<filename>',
                        help='Output script')

    parser.add_argument('-v', '--verbose', default=False, dest='verbose', action='store_true',
                        help='Enable verbose logging')
    parser.add_argument('--version', action='version', version=__version__)
    return parser


def _open_input(path):
    """The opened reader of a container input (inputs.READERS: Matroska, MP4, Ogg, AVI, transport or program stream), which also
    gives its script, chapters and streams; None for a WAV, FLAC, raw TrueHD (.thd), WavPack (.wv), TTA (.tta), Monkey's
    Audio (.ape), TAK (.tak) or MPEG audio (.mp2, .mpa, .m2a) input,
    which WavStream reads.  Any other extension, or a container's that does not open as one, is refused where the
    reference would have ffmpeg demux it."""
    ext = get_extension(path)
    fmt = next((f for f in READERS if ext in f.extensions), None)
    refusal = '{0}: demuxing is not supported, convert the input to WAV or FLAC first'.format(path)
    if fmt is None:
        raise SushiError(refusal)
    if fmt.opens_as is None:
        if fmt.name in ('WavPack', 'TTA', 'APE', 'TAK', 'MPEG audio'):
            fmt.reader(path)                       # its refusals, before the GPU is touched
        return None
    try:
        return fmt.reader(path)
    except (OSError, SushiError) as e:
        raise SushiError('{0} (it does not open as {1}: {2})'.format(refusal, fmt.opens_as, e))


def _select_audio(reader, idx, ffmpeg_audio=False):
    """The stream id of a container input's audio track (None for the other inputs), refusing what cannot be decoded
    and, with --ffmpeg-audio, what FFmpeg decodes to S32."""
    if reader is None:
        return None
    audio = reader.select_audio(idx)
    if ffmpeg_audio:
        swr.check(audio)
    return audio.id


def run(args):
    """sushi.py:528-736.  Everything up to the shift_script call is validation and small text files; nothing before
    it touches the GPU."""
    ignore_chapters = args.chapters_file is not None and args.chapters_file.lower() == 'none'

    check_file_exists(args.source, 'Source')
    check_file_exists(args.destination, 'Destination')
    check_file_exists(args.src_timecodes, 'Source timecodes')
    check_file_exists(args.dst_timecodes, 'Source timecodes')     # sic: the reference's title (sushi.py:540)
    check_file_exists(args.script_file, 'Script')
    if not ignore_chapters:
        check_file_exists(args.chapters_file, 'Chapters')
    if args.src_keyframes not in ('auto', 'make'):
        check_file_exists(args.src_keyframes, 'Source keyframes')
    if args.dst_keyframes not in ('auto', 'make'):
        check_file_exists(args.dst_keyframes, 'Destination keyframes')

    if (args.src_timecodes and args.src_fps) or (args.dst_timecodes and args.dst_fps):
        raise SushiError('Both fps and timecodes file cannot be specified at the same time')

    # where the reference opens the inputs with ffmpeg (sushi.py:553-554)
    src_mkv = _open_input(args.source)
    try:
        dst_mkv = _open_input(args.destination)
    except SushiError:
        if src_mkv:
            src_mkv.close()
        raise
    written = []
    try:
        return _run(args, ignore_chapters, src_mkv, dst_mkv, written)
    finally:
        for m in (src_mkv, dst_mkv):
            if m:
                m.close()
        if args.cleanup:
            for path in written:
                if os.path.exists(path):
                    os.remove(path)


def _run(args, ignore_chapters, src_mkv, dst_mkv, written):
    src_track = _select_audio(src_mkv, args.src_audio_idx, args.ffmpeg_audio)
    dst_track = _select_audio(dst_mkv, args.dst_audio_idx, args.ffmpeg_audio)
    # files taken out of the inputs, written once every check has passed: (path, function giving the text); and per
    # Matroska input, the tracks one walk over its clusters reads: (frames read, block times only)
    extract = []
    walks = [(m, [t], []) for m, t in ((src_mkv, src_track), (dst_mkv, dst_track)) if m is not None]

    def read_with_audio(mkv, payload=None, times=None):
        for m, p, t in walks:
            if m is mkv:
                p += [payload] if payload is not None else []
                t += [times] if times is not None else []

    if args.script_file:
        src_script_path = args.script_file
    elif src_mkv is not None:
        script_track = src_mkv.select('subtitles', args.src_script_idx)
        src_script_path = format_full_path(args.temp_dir, args.source, '.sushi' + script_track.script_type)
        extract.append((src_script_path, lambda: src_mkv.script_text(script_track)))
        read_with_audio(src_mkv, payload=script_track.id)
    else:
        raise SushiError("Script file isn't specified")

    if (args.src_keyframes and not args.dst_keyframes) or (args.dst_keyframes and not args.src_keyframes):
        raise SushiError('Either none or both of src and dst keyframes should be provided')

    create_directory_if_not_exists(args.temp_dir)

    script_extension = get_extension(src_script_path)
    if script_extension not in ('.ass', '.srt'):
        raise SushiError('Unknown script type')

    if args.output_script:
        dst_script_path = args.output_script
        dst_script_extension = get_extension(args.output_script)
        if dst_script_extension != script_extension:
            raise SushiError("Source and destination script file types don't match ({0} vs {1})"
                             .format(script_extension, dst_script_extension))
    else:
        dst_script_path = format_full_path(args.temp_dir, args.destination, '.sushi' + script_extension)

    if args.grouping and not ignore_chapters and args.chapters_file:
        if get_extension(args.chapters_file) == '.xml':
            chapter_times = get_xml_start_times(args.chapters_file)
        else:
            chapter_times = get_ogm_start_times(args.chapters_file)
    elif args.grouping and not ignore_chapters and src_mkv is not None:
        # the source's own chapters, also written out as OGM as the reference does (chapters.py:35-37)
        chapter_times = src_mkv.chapters
        extract.append((format_full_path(args.temp_dir, args.source, '.sushi.chapters.txt'), lambda: ''.join(
            'CHAPTER{0:02}={1}\nCHAPTER{0:02}NAME=\n'.format(i + 1, format_srt_time(t).replace(',', '.'))
            for i, t in enumerate(chapter_times))))
    else:
        chapter_times = []

    keyframes = None
    if args.src_keyframes:
        def select_keyframes(file_arg, path, mkv):
            if file_arg in ('auto', 'make'):
                auto_file = format_full_path(args.temp_dir, path, '.sushi.keyframes.txt')
                if file_arg == 'make' or not os.path.exists(auto_file):
                    if mkv is None or not mkv.streams('video'):
                        raise SushiError("Cannot make keyframes for {0} because it doesn't have any video!".format(path))
                    raise SushiError('Cannot make keyframes for {0}: making keyframes (SCXvid) is not supported, '
                                     'pass a keyframes file'.format(path))
                return auto_file
            return file_arg

        def select_timecodes(external_file, fps_arg, path, mkv):
            if external_file:
                return external_file
            if fps_arg:
                return None
            if mkv is not None and mkv.no_timecodes:
                raise SushiError('{0}: video timestamps cannot be read from {1} here; pass --src-fps / --dst-fps or a '
                                 'timecodes file'.format(path, mkv.no_timecodes))
            if mkv is not None and mkv.streams('video'):
                out = format_full_path(args.temp_dir, path, '.sushi.timecodes.txt')
                extract.append((out, mkv.timecodes_text))
                read_with_audio(mkv, times=mkv.streams('video')[0].id)
                return out
            raise SushiError('Fps, timecodes or video files must be provided if keyframes are used')

        src_keyframes_file = select_keyframes(args.src_keyframes, args.source, src_mkv)
        dst_keyframes_file = select_keyframes(args.dst_keyframes, args.destination, dst_mkv)
        src_timecodes_file = select_timecodes(args.src_timecodes, args.src_fps, args.source, src_mkv)
        dst_timecodes_file = select_timecodes(args.dst_timecodes, args.dst_fps, args.destination, dst_mkv)

    # every check has passed: one walk per Matroska input reads its audio, script and video times; the side products
    # are written from it, and the audio stays in memory for WavStream
    for mkv, payload_ids, time_ids in walks:
        mkv.prefetch(payload_ids, time_ids)
    for path, make in extract:
        text = make()
        written.append(path)
        with io.open(path, 'w', encoding='utf-8', newline='') as f:
            f.write(text)

    if args.src_keyframes:
        keyframes = load_keyframe_times(src_keyframes_file, dst_keyframes_file, args.src_fps, args.dst_fps,
                                        src_timecodes_file, dst_timecodes_file)

    tracks = {} if src_track is None and dst_track is None else dict(src_track=src_track, dst_track=dst_track)
    if args.ffmpeg_audio:
        tracks['ffmpeg_audio'] = True
    src = args.source if src_mkv is None else src_mkv
    dst = args.destination if dst_mkv is None else dst_mkv
    return shift_script(src, dst, src_script_path, dst_script_path,
                        sample_rate=args.sample_rate, sample_type=args.sample_type, chapter_times=chapter_times,
                        window=args.window, max_window=args.max_window, rewind_thresh=args.rewind_thresh,
                        grouping=args.grouping, smooth_radius=args.smooth_radius,
                        max_ts_duration=args.max_ts_duration, max_ts_distance=args.max_ts_distance,
                        keyframes=keyframes, max_kf_distance=args.max_kf_distance, kf_mode=args.kf_mode, **tracks)


def main(argv=None):
    """Parse `argv` (default sys.argv[1:]) and run.  Returns 0 on success and 2 after logging a
    SushiError, the reference's exit code; argparse exits 2 on bad flags by itself."""
    argv = sys.argv[1:] if argv is None else list(argv)
    args = create_arg_parser().parse_args(argv)
    handler = logging.StreamHandler()
    handler.setFormatter(logging.Formatter('%(message)s'))
    root = logging.getLogger()
    old_level = root.level
    root.addHandler(handler)
    root.setLevel(logging.DEBUG if args.verbose else logging.INFO)
    try:
        logging.info("Sushi's running with arguments: {0}".format(
            ' '.join(a if ' ' not in a else '"{0}"'.format(a) for a in argv)))
        start_time = time.time()
        run(args)
        logging.info('Done in {0}s'.format(time.time() - start_time))
        return 0
    except SushiError as e:
        logging.critical(str(e))
        return 2
    finally:
        root.removeHandler(handler)
        root.setLevel(old_level)
