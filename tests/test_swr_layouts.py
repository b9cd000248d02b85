"""What each reader says FFmpeg's decoder outputs (common.Audio's `fmt` and `layout`, for --ffmpeg-audio) against what
FFmpeg's decoder does output: every audio stream of the files the case writers make is opened with libavformat, its
packets are decoded with libavcodec until a frame comes out, and that frame's format and the decoder context's
`ch_layout` option are read.  A layout FFmpeg leaves unspecified is the default layout of its channel count, as the
ffmpeg command line assumes.  A reader that cannot tell the format before decoding (None: BD-LPCM, WavPack in
Matroska) or has no layout for a channel count is not compared; the stage refuses those streams."""
import ctypes

import pytest

from oracle import ref_flac
from sushi_b200 import SushiError, inputs
from tests import flac_cases, mkv_alac_cases, mkv_cases, mkv_tta_cases, mkv_wavpack_cases, mp4_cases
from tests import ref_mp4, ts_cases, tta_cases, wavpack_cases

S16, S16P, S32, S32P = 1, 6, 2, 7
FMT = {S16: 'S16', S16P: 'S16', S32: 'S32', S32P: 'S32'}
COMPARED = set()


def ffmpeg_audio(path):
    """{stream id: (sample format, channel mask)} of each audio stream FFmpeg decodes a frame of"""
    fmt, codec, util = ref_flac.libs()
    streams = ref_mp4.demux(path, packets=False).streams
    out = {}
    for sid, (kind, _, _) in enumerate(streams):
        if kind != 'audio':
            continue
        ctx = ref_mp4._open(path)
        dec = pkt = frame = ctypes.c_void_p()
        try:
            fmt.avformat_find_stream_info(ctx, None)
            par = ref_mp4._ptr(ref_mp4._ptr(ref_mp4._ptr(ctx.value + 48) + 8 * sid) + 16)
            c = codec.avcodec_find_decoder(ref_mp4._i32(par + 4))
            if not c:
                continue
            dec = ctypes.c_void_p(codec.avcodec_alloc_context3(c))
            if codec.avcodec_parameters_to_context(dec, par) < 0 or codec.avcodec_open2(dec, c, None) < 0:
                continue
            pkt = ctypes.c_void_p(codec.av_packet_alloc())
            frame = ctypes.c_void_p(util.av_frame_alloc())
            got = False
            while not got and fmt.av_read_frame(ctx, pkt) >= 0:
                if ref_mp4._i32(pkt.value + 36) == sid:
                    codec.avcodec_send_packet(dec, pkt)
                    got = codec.avcodec_receive_frame(dec, frame) == 0
                codec.av_packet_unref(pkt)
            if not got:
                continue
            out[sid] = (FMT.get(ref_mp4._i32(frame.value + 116)),) + ref_mp4.decoder_layout(dec)   # AVFrame.format
        finally:
            if frame:
                util.av_frame_free(ctypes.byref(frame))
            if pkt:
                codec.av_packet_free(ctypes.byref(pkt))
            if dec:
                codec.avcodec_free_context(ctypes.byref(dec))
            fmt.avformat_close_input(ctypes.byref(ctx))
    return out


def compare(path):
    """-> number of streams compared; asserts every one agrees"""
    seen = 0
    theirs = ffmpeg_audio(path)
    reader, _ = inputs.open_input(path)
    try:
        for sid, (fmt, mask, channels) in theirs.items():
            try:
                audio = reader.select_audio(sid if hasattr(reader, 'tracks') or hasattr(reader, 'select') else None)
            except SushiError:
                continue
            if audio.fmt is None:
                continue
            assert audio.fmt == fmt, (path, sid, audio.fmt, fmt)
            if fmt == 'S16' and channels in (audio.layout or {}):
                assert audio.layout[channels] == mask, (path, sid, hex(audio.layout[channels]), hex(mask))
                seen += 1
                COMPARED.add((audio.label or 'PCM', channels))
    finally:
        if hasattr(reader, 'close'):
            reader.close()
    return seen


def write(tmp_path, name, data):
    path = tmp_path / name
    path.write_bytes(data)
    return str(path)


def test_flac(tmp_path):
    n = sum(compare(write(tmp_path, c.name + '.flac', c.flac)) for c in flac_cases.named_cases() if c.bits == 16)
    assert n >= 3


def test_tta(tmp_path):
    n = sum(compare(write(tmp_path, c.name + '.tta', c.tta())) for c in tta_cases.all_cases() if c.bits == 16)
    assert n >= 1


def test_wavpack(tmp_path):
    n = sum(compare(write(tmp_path, c.name + '.wv', c.wv())) for c in wavpack_cases.all_cases() if c.bits == 16)
    assert n >= 1


def test_matroska(tmp_path):
    cases = [c for c in mkv_cases.audio_cases()] + [m for m, _ in mkv_alac_cases.cases()] + \
        [m for m, _, how in mkv_tta_cases.cases() if how == 'decoded'] + [c[0] for c in mkv_wavpack_cases.cases()]
    n = sum(compare(write(tmp_path, c.name + '.mka', c.data)) for c in cases)
    assert n >= 3


def test_mp4(tmp_path):
    n = sum(compare(c.write(tmp_path)) for c in mp4_cases.good_cases())
    assert n >= 1


@pytest.mark.parametrize('case', ts_cases.all_cases()[:3], ids=lambda c: c.name)
def test_transport_stream_formats_are_left_to_the_decoder(tmp_path, case):
    reader, _ = inputs.open_input(case.write(tmp_path))
    try:
        audio = reader.select_audio(None)
    except SushiError:
        return
    finally:
        reader.close()
    assert audio.fmt in (None, 'S32')


def test_what_was_compared():
    print('codec and channel count compared:', sorted(COMPARED))
