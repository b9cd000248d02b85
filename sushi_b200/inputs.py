"""The input formats, in one table.  Each has a host-side reader in its own module (this is the only module that knows
them all) with one method, select_audio(track=None), which makes every refusal that needs no GPU and returns the
common.Audio WavStream loads.  WavStream detects the format (open_input); the command line goes by file extension."""
import collections

from . import ape, avi, matroska, mp4, mpa, mpegps, mpegts, ogg, tak, truehd, tta, wavpack
from .flac import FlacFile, is_flac
from .wav import DownmixedWavFile

# name: as the log names it; extensions: what the command line takes it by; sniff(path): whether a file is one (by its
# content; a transport stream, a program stream, raw MPEG audio and a TrueHD stream by its name), asked in the table's order; reader: its class; opens_as:
# for a container, whose script, chapters and streams the command line reads too, what its extensions must open as.
Format = collections.namedtuple('Format', 'name extensions sniff reader opens_as')
FORMATS = (
    Format('transport stream', mpegts.TS_EXTENSIONS, mpegts.is_transport_stream, mpegts.TransportStream,
           'a transport stream'),
    Format('MP4', mp4.MP4_EXTENSIONS, mp4.is_mp4, mp4.Mp4File, 'an MP4 file'),
    Format('Matroska', matroska.MATROSKA_EXTENSIONS, matroska.is_matroska, matroska.MatroskaFile, 'a Matroska file'),
    Format('TrueHD', truehd.THD_EXTENSIONS, truehd.is_truehd, truehd.TrueHDFile, None),
    Format('WavPack', wavpack.WV_EXTENSIONS, wavpack.is_wavpack, wavpack.WavPackFile, None),
    Format('TTA', tta.TTA_EXTENSIONS, tta.is_tta, tta.TTAFile, None),
    Format('FLAC', ('.flac',), is_flac, FlacFile, None),
    Format('WAV', ('.wav',), lambda path: True, DownmixedWavFile, None),      # whatever is nothing else
)
# The MPEG systems whose audio is MP2: program streams and raw MPEG audio, both known by their names.  They are asked
# before the table above.
MPEG_FORMATS = (
    Format('program stream', mpegps.PS_EXTENSIONS, mpegps.is_program_stream, mpegps.ProgramStream,
           'a program stream'),
    Format('MPEG audio', mpa.MPA_EXTENSIONS, mpa.is_mpeg_audio, mpa.MpegAudioFile, None),
)
# Ogg files, known by their capture pattern, asked after those and before the table above
OGG_FORMATS = (
    Format('Ogg', ogg.OGG_EXTENSIONS, ogg.is_ogg, ogg.OggFile, 'an Ogg file'),
)
# Monkey's Audio files, known by their `MAC ` marker (after an optional ID3v2 tag), asked after those and before the
# table above
APE_FORMATS = (
    Format('APE', ape.APE_EXTENSIONS, ape.is_ape, ape.ApeFile, None),
)
# TAK files, known by their `tBaK` marker (after an optional ID3v2 tag), asked after those and before the table above
TAK_FORMATS = (
    Format('TAK', tak.TAK_EXTENSIONS, tak.is_tak, tak.TakFile, None),
)
# AVI files, known by `RIFF` + size + `AVI `, asked after those and before the table above (whose WAV reader takes every
# other RIFF file)
AVI_FORMATS = (
    Format('AVI', avi.AVI_EXTENSIONS, avi.is_avi, avi.AviFile, 'an AVI file'),
)
# READERS is the whole table, in the order open_input asks.
READERS = MPEG_FORMATS + OGG_FORMATS + APE_FORMATS + TAK_FORMATS + AVI_FORMATS + FORMATS


def open_input(source):
    """(reader, format name) of `source`: a file name, whose format is detected by content, or an opened container
    reader (MatroskaFile, Mp4File, TransportStream, ProgramStream, OggFile, AviFile), which is returned as it is and never
    sniffed."""
    for f in READERS:
        if f.opens_as and isinstance(source, f.reader):
            return source, f.name
    for f in READERS:
        if f.sniff(source):
            return f.reader(source), f.name
