"""Load time of each input format on one GPU, against the loads it is compared with.

    python tools/load.py FORMAT [FORMAT ...] [--minutes M ...] [--bits B ...] [--runs 3] [--dir /tmp]

FORMAT is one of the names in FORMATS below.  For each format and each length and depth (its defaults, or --minutes
and --bits), the tool writes 48 kHz stereo files of that length, loads each once untimed (page cache, device pool),
then alternates the timed loads `--runs` times and prints one JSON line per load: what was loaded, file bytes, wall ms
of WavStream(path) from one device synchronise to the next, and device ms per kernel class from sb_profile_*.  Each
format's lines start with a row naming the card (name, power limit, SM clock, maximum SM clock, memory clock) and its
SM count, and end with `card_after`, read again.  Files go to a temporary directory (or --dir) and are removed as soon
as they have been measured.  Nothing is asserted."""
import argparse
import collections
import ctypes
import json
import os
import pathlib
import shutil
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from sushi_b200 import _native, matroska, mp4, mpegts, tta, wavpack  # noqa: E402
from sushi_b200.wavstream import FlacFile, WavStream  # noqa: E402
from tests import (alac_cases, ape_cases, avi_cases, flac_cases as fc, loader_cases as lc, mkv_cases, mp2_cases,  # noqa
                   mp4_cases, ogg_cases, ps_cases, ref_mp2, ref_swr, tak_cases, truehd_cases, ts_cases, tta_cases,
                   wavpack_cases)


# ---- what every format shares ------------------------------------------------------------------------------------

def card():
    """One read-only nvidia-smi query: name, power limit, SM clock, maximum SM clock, memory clock."""
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def sm_count():
    try:
        import torch
        return torch.cuda.get_device_properties(_native.bound_device() or 0).multi_processor_count
    except Exception:
        return None


def kernel_ms(lib):
    """Device ms per kernel class since the last sb_profile_reset."""
    phases = {}
    for name in lib.sb_profile_names().decode().split(','):
        if not name:
            continue
        ms, n = ctypes.c_double(), ctypes.c_int64()
        lib.sb_profile_get(name.encode(), ctypes.byref(ms), ctypes.byref(n))
        if n.value:
            phases[name] = round(ms.value, 3)
    return phases


def load_once(lib, path, ffmpeg_audio=False):
    """(seconds, device ms per kernel class) of one WavStream(path): the window opens and closes on a device
    synchronise, so it holds the whole load and nothing else."""
    lib.sb_profile_reset()
    _native.check(lib.sb_sync(), 'sb_sync')
    t0 = time.perf_counter()
    s = WavStream(path, 12000, 'uint8', ffmpeg_audio=ffmpeg_audio)
    _native.check(lib.sb_sync(), 'sb_sync')
    wall = time.perf_counter() - t0
    phases = kernel_ms(lib)
    s.close()
    return wall, phases


def pcm_bytes(pcm, width):
    if width == 2:
        return pcm.astype('<i2').tobytes()
    u = (pcm.reshape(-1) & 0xFFFFFF).astype(np.uint32)
    return np.stack([u & 0xFF, (u >> 8) & 0xFF, u >> 16], 1).astype(np.uint8).tobytes()


def write(path, data):
    with open(path, 'wb') as f:
        f.write(data)
    return path


def write_repeated(path, head, one, reps, rest):
    with open(path, 'wb') as f:
        f.write(head)
        for _ in range(reps):
            f.write(one)
        f.write(rest)
    return path


def write_wav(path, pcm, reps, tail, width):
    """The 48 kHz stereo WAV of PCM block `pcm` repeated `reps` times, then `tail`."""
    one, rest = pcm_bytes(pcm, width), pcm_bytes(tail, width)
    return write_repeated(path, lc.riff(2, 48000, width, b'', len(one) * reps + len(rest)), one, reps, rest)


def sized(fields, *files):
    """[(row fields, path)]: `fields` with each file's input kind and bytes."""
    return [(dict(fields, input=kind, bytes=os.path.getsize(path)), path) for kind, path in files]


FLAC_BLOCK = 4608
FLAC_SPEC = dict(kind='lpc', order=10, precision=13, porder=6, porder_search=True, method='rice')


def coded(j):
    """The channel assignment of FLAC frame j: mid/side (10) on one frame in four, independent (1) on the rest."""
    return 10 if j % 4 == 0 else 1


def write_flac(directory, minutes, bits):
    """The FLAC file other formats are compared with: every frame LPC order 10, coefficient precision 13, Rice
    partitions up to order 6 chosen per frame, mid/side on one frame in four; the PCM repeats every 256 frames, which
    the decoder does not know.  -> (path, the repeated PCM, its repetitions, the PCM after them)"""
    n = minutes * 60 * 48000
    period = 1024 * 1152 // FLAC_BLOCK
    frames, tail = n // FLAC_BLOCK, n % FLAC_BLOCK or 100
    data, base, tail_pcm = fc.periodic_file(frames, tail, bits, coded, 11, 48000, FLAC_BLOCK, period,
                                            FLAC_SPEC, parts=True)
    path = write(os.path.join(directory, 'a%d_%d.flac' % (minutes, bits)), data)
    return path, base, frames // period, np.concatenate([base[:(frames % period) * FLAC_BLOCK], tail_pcm])


def plain_read(path):
    """The file read as WavStream reads a transport stream: chunks of mpegts.CHUNK_BYTES into one page-locked
    buffer."""
    buf = _native.pinned_empty((mpegts.CHUNK_BYTES,), np.uint8)
    view = memoryview(buf)
    t = time.perf_counter()
    n = 0
    with open(path, 'rb', buffering=0) as f:
        while True:
            got = f.readinto(view)
            if not got:
                break
            n += got
    return {'bytes_read': n, 'wall_ms': round(1e3 * (time.perf_counter() - t), 1), 'kernel_ms': {}}


def mkv_walk(path):
    """The container walk alone: MatroskaFile and the frames of its audio track."""
    t0 = time.perf_counter()
    with matroska.MatroskaFile(path) as f:
        table = f.frames([f.select('audio', None).id])[1]
        read = f.bytes_read
    return {'host_ms': round(1e3 * (time.perf_counter() - t0), 1), 'bytes_read': read, 'audio_frames': len(table)}


def mp4_reader(path):
    t0 = time.perf_counter()
    with mp4.Mp4File(path) as f:
        t1 = time.perf_counter()
        table = f.frames(f.select('audio', None))
        t2 = time.perf_counter()
        return {'reader': {'open_ms': round(1e3 * (t1 - t0), 1), 'table_ms': round(1e3 * (t2 - t1), 1),
                           'bytes_read': f.bytes_read, 'samples': len(table)}}


def wavpack_walk(path):
    t0 = time.perf_counter()
    f = wavpack.WavPackFile(path)
    return {'host': {'walk_ms': round(1e3 * (time.perf_counter() - t0), 1), 'blocks': len(f.table)}}


def tta_walk(path):
    t0 = time.perf_counter()
    f = tta.TTAFile(path)
    return {'host': {'walk_ms': round(1e3 * (time.perf_counter() - t0), 1), 'frames': len(f.offsets)}}


# input kind -> leg(path): the row fields of a timed leg that replaces the load
LEGS = {'plain_read': plain_read, 'mkv_walk': mkv_walk}
# input kind -> probe(path): row fields the host side measures after each load of that kind
PROBES = {'alac': mp4_reader, 'wavpack': wavpack_walk, 'tta': tta_walk}


# ---- the formats: each builder writes one case's files and returns [(row fields, path)] in the order the timed runs
# alternate them ----------------------------------------------------------------------------------------------------

def build_flac(directory, minutes, bits):
    flac, base, reps, rest = write_flac(directory, minutes, bits)
    wav = write_wav(os.path.join(directory, 'a%d_%d.wav' % (minutes, bits)), base, reps, rest, bits // 8)
    return sized({'minutes': minutes, 'bits': bits}, ('flac', flac), ('wav', wav))


MKV_BLOCK, MKV_PERIOD, MKV_FPS = 4096, 256, 24000 / 1001.0
MKV_RATES = {(24, None): 40.0, (90, None): 8.0}           # video Mbit/s: about 7 GB and 5.5 GB


def flac_frame_slices(data, n_frames):
    """(the header blocks, every frame) of a periodic_file: the payloads repeat every MKV_PERIOD frames, so the lengths
    of the first MKV_PERIOD frames (found by their exact headers) give every offset."""
    first = FlacFile.from_bytes(data[:65536], 'audio').frame_offset
    heads = [fc.frame_header(i, MKV_BLOCK, 48000, 2, coded(i % MKV_PERIOD), 16, {})[0]
             for i in range(MKV_PERIOD + 1)]
    at, payload = first, []
    for i in range(MKV_PERIOD):
        nxt = data.index(heads[i + 1], at + len(heads[i]))
        payload.append(nxt - at - len(heads[i]))
        at = nxt
    view = memoryview(data)
    frames, at = [], first
    for i in range(n_frames):
        n = len(fc.frame_header(i, MKV_BLOCK, 48000, 2, coded(i % MKV_PERIOD), 16, {})[0]) + payload[i % MKV_PERIOD]
        frames.append(view[at:at + n])
        at += n
    frames.append(view[at:])
    return data[:first], frames


def read_through(path):
    """Read the whole file once (the page cache keeps what it can); returns the seconds it took."""
    t0 = time.perf_counter()
    with open(path, 'rb', buffering=0) as f:
        while f.read(64 << 20):
            pass
    return time.perf_counter() - t0


def build_mkv(directory, minutes, bits, mbps=None):
    """A remux-shaped MKV: a 16-bit FLAC track (4096-sample frames, one per block) beside 23.976 fps video of random
    bytes at `mbps`, and the .flac file of the same audio.  Free space is checked first.  Both files are read through
    once, so that the MKV's video pages are cached too (a load reads only their block headers); before each pair of
    loads the container walk is timed alone."""
    mbps = mbps or MKV_RATES[minutes, bits]
    need = minutes * 60 * (mbps * 1e6 / 8 + 2 * 100000)           # video + MKV and FLAC audio
    free = shutil.disk_usage(directory).free
    if free < 1.2 * need:
        sys.exit('load.py mkv: %.1f GB free in %s, %.1f GB needed' % (free / 1e9, directory, 1.2 * need / 1e9))
    t0 = time.perf_counter()
    n = minutes * 60 * 48000
    n_frames, tail = n // MKV_BLOCK, n % MKV_BLOCK or 100
    data, _ = fc.periodic_file(n_frames, tail, 16, coded, 11, 48000, MKV_BLOCK, MKV_PERIOD, FLAC_SPEC)
    flac = write(os.path.join(directory, 'a%d.flac' % minutes), data)
    private, frames = flac_frame_slices(data, n_frames)
    mkv = os.path.join(directory, 'a%d.mkv' % minutes)
    video = int(minutes * 60 * MKV_FPS)
    _, vbytes = mkv_cases.write_av(mkv, private, frames, [MKV_BLOCK] * n_frames + [tail], 48000, 2, 16, video,
                                   int(mbps * 1e6 / 8 / MKV_FPS), 12)
    sizes = {'mkv': os.path.getsize(mkv), 'flac': os.path.getsize(flac)}
    print(json.dumps({'audio_frames': n_frames + 1, 'video_frames': video, 'video_bytes': vbytes, 'minutes': minutes,
                      'mbps': mbps, 'bytes': sizes, 'build_s': round(time.perf_counter() - t0, 1)}), flush=True)
    print(json.dumps({'minutes': minutes, 'read_through_s': {k: round(read_through(p), 2) for k, p in
                                                              (('mkv', mkv), ('flac', flac))}}), flush=True)
    return [({'minutes': minutes, 'input': 'mkv_walk'}, mkv)] + sized({'minutes': minutes}, ('mkv', mkv),
                                                                       ('flac', flac))


def build_truehd(directory, minutes, bits):
    """One restart segment of 64 AUs of 16-bit programme material (FIR / IIR prediction, Huffman codebooks, quant
    steps, matrices) repeated, the WAV of the same samples, and write_flac's 16-bit file of the same length (other
    audio of the same shape)."""
    rng = np.random.default_rng([truehd_cases.SEED, 70])
    pcm = truehd_cases.make_pcm(64 * 40, 2, 16, 48000, rng)
    style = {'permute': False, 'filters': True, 'huff': True, 'quant': True, 'matrix': True, 'omit': True}
    seg = truehd_cases.periodic_segment(pcm, 16, n_sub=1, style=style, seed=71)
    reps = minutes * 60 * 48000 // (64 * 40)
    thd = write_repeated(os.path.join(directory, 'a%d.thd' % minutes), b'', seg, reps, b'')
    wav = write_wav(os.path.join(directory, 'a%d.wav' % minutes), pcm >> 8, reps, pcm[:0], 2)
    flac = write_flac(directory, minutes, 16)[0]
    files = sized({'minutes': minutes}, ('truehd', thd), ('wav', wav), ('flac', flac))
    sms = sm_count()
    files[0][0].update(segments=reps, threads_per_sm=round(reps / sms, 1) if sms else None)
    return files


# video filler packets per second by (minutes, bits): about 40 Mbit/s and 10 Mbit/s in all
TS_FILLER = {(24, 16): 25152, (24, 24): 24752, (90, 16): 5440, (90, 24): 5040}


def build_ts(directory, minutes, bits, video=None):
    """A BDAV stream of LPCM (tests/ts_cases.py long_m2ts: one second of 240-frame PES packets and `video` filler
    packets, repeated) and the WAV of the same PCM; the .m2ts is also read plainly, as WavStream reads it."""
    video = video or TS_FILLER[minutes, bits]
    m2ts = os.path.join(directory, 'a%d_%d.m2ts' % (minutes, bits))
    pcm, reps = ts_cases.long_m2ts(m2ts, minutes, bits=bits, video_packets=video)
    wav = ts_cases.write_wav(os.path.join(directory, 'a%d_%d.wav' % (minutes, bits)), np.tile(pcm, (reps, 1)), 48000)
    mbps = os.path.getsize(m2ts) * 8 / 1e6 / (os.path.getsize(wav) / 192000.0)
    files = sized({'file': '%d min %d-bit LPCM' % (minutes, bits), 'mbit_s': round(mbps, 1)}, ('m2ts', m2ts),
                  ('wav', wav), ('plain_read', m2ts))
    for row, _ in files[:2]:
        row['bytes_read'] = row['bytes']                           # a load reads the whole file
    return files


def build_alac(directory, minutes, bits):
    """An .m4a of Apple's default coding (pb 40, mb 10, kb 14, frames of 4096, LPC order 8; 24-bit samples with one
    shifted byte): 16 frames repeated; the WAV of the same samples; and write_flac's file (other audio of the same
    shape)."""
    cfg, frames, pcm, _ = alac_cases.long_stream(bits=bits, minutes=minutes, n_unique=16)
    reps = minutes * 60 * 48000 // (len(frames) * cfg.frame_length)
    case = alac_cases.AlacCase('a', cfg, frames * reps, pcm[:0], set())
    case.pcm = pcm
    m4a = write(os.path.join(directory, 'alac%d_%d.m4a' % (minutes, bits)),
                mp4_cases.build('a', [mp4_cases.alac_trak(case, per_chunk=(64,), edits=None)], ftyp=b'M4A '))
    wav = write_wav(os.path.join(directory, 'alac%d_%d.wav' % (minutes, bits)), pcm, reps, pcm[:0], bits // 8)
    flac = write_flac(directory, minutes, bits)[0]
    return sized({'minutes': minutes, 'bits': bits}, ('alac', m4a), ('flac', flac), ('wav', wav))


def build_wavpack(directory, minutes, bits):
    """tests/wavpack_cases.py's long stream (4 blocks of 0.5 s, joint stereo, 4 decorrelation terms, repeated), the
    WAV of the same samples, and write_flac's file (other audio of the same shape)."""
    case, data, reps = wavpack_cases.long_stream(bits=bits, minutes=minutes)
    wv = write(os.path.join(directory, 'wv%d_%d.wv' % (minutes, bits)), data)
    del data
    wav = write_wav(os.path.join(directory, 'wv%d_%d.wav' % (minutes, bits)), case.pcm, reps, case.pcm[:0], bits // 8)
    flac = write_flac(directory, minutes, bits)[0]
    return sized({'minutes': minutes, 'bits': bits}, ('wavpack', wv), ('flac', flac), ('wav', wav))


def build_tta(directory, minutes, bits):
    """tests/tta_cases.py's long stream (one whole frame of 50 155 samples repeated, then a short one), the WAV of the
    same samples, and write_flac's file (other audio of the same shape)."""
    case, data, reps = tta_cases.long_stream(bits=bits, minutes=minutes)
    path = write(os.path.join(directory, 'tta%d_%d.tta' % (minutes, bits)), data)
    del data
    fl = case.frame_length
    wav = write_wav(os.path.join(directory, 'tta%d_%d.wav' % (minutes, bits)), case.pcm[:fl], reps, case.pcm[fl:],
                    bits // 8)
    flac = write_flac(directory, minutes, bits)[0]
    return sized({'minutes': minutes, 'bits': bits}, ('tta', path), ('flac', flac), ('wav', wav))


def build_ape(directory, minutes, bits):
    """tests/ape_cases.py's long stream (one insane-level frame of the size Monkey's Audio writes, 1 179 648 blocks,
    repeated), the WAV of the same samples, and write_flac's file (other audio of the same shape)."""
    case, data, reps = ape_cases.long_stream(bits=bits, minutes=minutes)
    path = write(os.path.join(directory, 'ape%d_%d.ape' % (minutes, bits)), data)
    del data
    wav = write_wav(os.path.join(directory, 'ape%d_%d.wav' % (minutes, bits)), case.pcm, reps, case.pcm[:0],
                    bits // 8)
    flac = write_flac(directory, minutes, bits)[0]
    return sized({'minutes': minutes, 'bits': bits, 'frame_blocks': case.bpf, 'frames': reps}, ('ape', path),
                 ('flac', flac), ('wav', wav))


def build_tak(directory, minutes, bits):
    """tests/tak_cases.py's long stream (one 250 ms frame at the largest filter order, repeated with its own frame
    numbers), the WAV of the same samples, and write_flac's file (other audio of the same shape)."""
    case, data, reps = tak_cases.long_stream(bits=bits, minutes=minutes)
    path = write(os.path.join(directory, 'tak%d_%d.tak' % (minutes, bits)), data)
    del data
    wav = write_wav(os.path.join(directory, 'tak%d_%d.wav' % (minutes, bits)), case.pcm, reps, case.pcm[:0],
                    bits // 8)
    flac = write_flac(directory, minutes, bits)[0]
    return sized({'minutes': minutes, 'bits': bits, 'frame_samples': case.nb, 'frames': reps}, ('tak', path),
                 ('flac', flac), ('wav', wav))


def build_avi(directory, minutes, bits):
    """tests/avi_cases.py's long OpenDML file: 1 s chunks of 48 kHz stereo PCM beside 4 kB chunks of random-byte video,
    RIFF AVI up to 1 GiB and RIFF AVIX lists after it."""
    path = os.path.join(directory, 'avi%d_%d.avi' % (minutes, bits))
    avi_cases.long_file(path, minutes, bits)
    return sized({'minutes': minutes, 'bits': bits}, ('avi (PCM)', path))


PS_PACK = 2048
PS_VIDEO_PER_AUDIO = 11              # video packs between audio packs: about 1.5 GB for 90 minutes


def build_ps(directory, minutes, bits):
    """A DVD-style program stream of 2048-byte packs: tests/mp2_cases.py's long MP2 stream (192 kbit/s) with video
    packs of random bytes (no zero byte, one off-chain pack start code each) between its packs."""
    frames, data = mp2_cases.long_stream(minutes)
    rng = np.random.default_rng([3])
    room = PS_PACK - 14 - 14                              # pack header, PES header with PTS
    video = bytearray(rng.integers(1, 256, room, dtype=np.uint8).tobytes())
    video[room // 2:room // 2 + 4] = b'\x00\x00\x01\xba'
    vpes = ps_cases.pes2(ps_cases.VIDEO, bytes(video), 90000)
    assert len(vpes) + 14 == PS_PACK and struct.unpack('>H', vpes[4:6])[0] == PS_PACK - 20
    path = os.path.join(directory, 'long.vob')
    scr = 0
    with open(path, 'wb') as f:
        for at in range(0, len(data), room):
            out = [ps_cases.pack_header(scr, True), ps_cases.pes2(ps_cases.AUDIO, data[at:at + room], 90000 + at)]
            for _ in range(PS_VIDEO_PER_AUDIO):
                scr += 300
                out += [ps_cases.pack_header(scr, True), vpes]
            f.write(b''.join(out))
        f.write(b'\x00\x00\x01\xb9')
    return sized({'minutes': minutes, 'frames': len(frames)}, ('mp2 (program stream)', path))


OGG_SERIAL = 0x0665
# The Ogg files DESIGN.md measured carry this comment, named after the script that first wrote them; it stays so that
# the files stay the same byte for byte.
OGG_ENCODER = b'ENCODER=tools/ogg_load.py'


def flac_frame_offsets(data, first):
    """The offsets of a FLAC file's frames: the sync codes whose coded frame number is the next one and whose header
    passes its CRC-8 (false syncs inside VERBATIM payloads are passed over)."""
    d = np.frombuffer(data, np.uint8)
    cand = np.flatnonzero((d[first:-1] == 0xFF) & (d[first + 1:] == 0xF8)) + first
    out, want = [], 0
    for c in cand.tolist():
        b = data[c + 4]
        extra = 0
        if b < 0x80:
            n = b
        else:
            extra = 1 if b < 0xE0 else 2 if b < 0xF0 else 3
            n = b & (0x3F >> extra)
            for k in range(extra):
                n = (n << 6) | (data[c + 5 + k] & 0x3F)
        bs, sr = data[c + 2] >> 4, data[c + 2] & 15
        hl = 5 + extra + {6: 1, 7: 2}.get(bs, 0) + {12: 1, 13: 2, 14: 2}.get(sr, 0)
        if n == want and fc.crc8(data[c:c + hl]) == data[c + hl]:
            out.append(c)
            want += 1
    return out + [len(data)]


def ogg_crcs(pages):
    """Ogg CRC-32 of each page (CRC field zero), vectorised across pages: leading zeros leave a CRC from 0 unchanged,
    so the pages are right-aligned in one array and folded a column at a time."""
    width = max(len(p) for p in pages)
    m = np.zeros((len(pages), width), np.uint8)
    for i, p in enumerate(pages):
        m[i, width - len(p):] = np.frombuffer(p, np.uint8)
    c = np.zeros(len(pages), np.uint32)
    for j in range(width):
        c = (c << np.uint32(8)) ^ ogg_cases.CRC_TABLE[(c >> np.uint32(24)) ^ m[:, j]]
    return c


def build_ogg(directory, minutes, bits):
    """24-bit FLAC (tests/flac_cases.py's periodic file: VERBATIM frames of 1152 samples, every 16th LPC) in Ogg pages
    as libFLAC's Ogg encoder lays them out, one frame per page."""
    data, _ = fc.periodic_file(minutes * 60 * 48000 // 1152, 500, 24, lambda j: None if j % 16 else 1, 11)
    first = 4
    while not data[first] & 0x80:
        first += 4 + int.from_bytes(data[first + 1:first + 4], 'big')
    first += 4 + int.from_bytes(data[first + 1:first + 4], 'big')
    offs = flac_frame_offsets(data, first)
    blocks = ogg_cases.split_blocks(data, first)
    info = bytes([blocks[0][0] & 0x7F]) + bytes(blocks[0][1:])
    mapping = b'\x7fFLAC\x01\x00' + struct.pack('>H', 1) + b'fLaC' + info
    comment = ogg_cases.vorbis_comment_block([OGG_ENCODER])
    comment[0] |= 0x80
    packets = [mapping, bytes(comment)] + [data[a:b] for a, b in zip(offs, offs[1:])]
    del data
    path = os.path.join(directory, 'long.oga')
    with open(path, 'wb') as f:
        for a in range(0, len(packets), 8192):
            raw = []
            for i, pk in enumerate(packets[a:a + 8192], a):
                lacing = [255] * (len(pk) // 255) + [len(pk) % 255]
                flags = (2 if i == 0 else 0) | (4 if i == len(packets) - 1 else 0)
                raw.append(b'OggS' + bytes([0, flags]) + struct.pack('<qII', 1152 * max(0, i - 1), OGG_SERIAL, i) +
                           b'\0\0\0\0' + bytes([len(lacing)]) + bytes(lacing) + pk)
            f.write(b''.join(p[:22] + struct.pack('<I', int(c)) + p[26:] for p, c in zip(raw, ogg_crcs(raw))))
    return sized({'minutes': minutes, 'frames': len(offs) - 1, 'pages': len(packets)},
                 ('flac 24-bit stereo (Ogg)', path))


def build_mp2(directory, minutes, bits):
    """tests/mp2_cases.py's long stream (120 random layer II frames at 192 kbit/s, cycled) in a Matroska file of one
    block per 100 frames."""
    frames, _ = mp2_cases.long_stream(minutes)
    sizes = [len(f) for f in frames]
    pieces = [sum(sizes[k:k + 100]) for k in range(0, len(sizes), 100)]
    case = mp2_cases.Case('long', frames, [mp2_cases.FrameSpec(mode=0, rate=48000)])
    path = mp2_cases.mkv_file('long', case, pieces).write(pathlib.Path(directory))
    return sized({'minutes': minutes, 'frames': len(frames)}, ('mp2 (Matroska)', path))


def ffmpeg_mp2(lib, minutes, runs):
    """FFmpeg's mp2 decoder (tests/ref_mp2.py) on one CPU core, on the frames of build_mp2's file, timed once."""
    frames, _ = mp2_cases.long_stream(minutes)
    t0 = time.perf_counter()
    pcm = ref_mp2.decode_packets(frames)[0]
    ms = round(1e3 * (time.perf_counter() - t0), 1)
    print(json.dumps({'ffmpeg_mp2_one_core_ms': ms, 'samples': int(pcm.shape[0])}), flush=True)


def build_swr(directory, minutes, bits):
    """write_flac's 16-bit file, loaded without and with --ffmpeg-audio."""
    flac = write_flac(directory, minutes, 16)[0]
    return [({'minutes': minutes, 'input': 'flac stereo', 'ffmpeg_audio': mode}, flac) for mode in (False, True)]


def swr_alone(lib, minutes, runs):
    """sb_pcm_swr alone (48 kHz -> 12 kHz) on stereo and on 5.1 noise already on the device: wall and swr_resample
    device ms, best of `runs` + 1; then libswresample's own host time on the same PCM (tests/ref_swr.py, FMA3 path,
    4096-frame feeds), what the reference's ffmpeg spends on this step."""
    for mask in (0x3, 0x3f):
        channels = bin(mask).count('1')
        rng = np.random.default_rng(minutes * mask)
        pcm = (rng.standard_normal((minutes * 60 * 48000, channels), np.float32) * 6000).astype(np.int16)
        h = _native.decode(None, 'sb_pcm_from_le', pcm.ctypes.data_as(ctypes.c_void_p), len(pcm), channels, 2, 48000)
        best = None
        try:
            for _ in range(runs + 1):
                lib.sb_profile_reset()
                out = ctypes.c_void_p()
                t0 = time.perf_counter()
                _native.check(lib.sb_pcm_swr(h, mask, 12000, ctypes.byref(out)), 'sb_pcm_swr')
                wall = time.perf_counter() - t0
                lib.sb_pcm_destroy(out)
                k = kernel_ms(lib).get('swr_resample')
                if best is None or wall < best[0]:
                    best = (wall, k)
        finally:
            lib.sb_pcm_destroy(h)
        t0 = time.perf_counter()
        ref_swr.convert(pcm, mask, 48000, 12000)
        host = time.perf_counter() - t0
        print(json.dumps({'minutes': minutes, 'layout': hex(mask), 'sb_pcm_swr_wall_ms': round(1e3 * best[0], 2),
                          'swr_resample_ms': best[1], 'libswresample_host_s': round(host, 2)}), flush=True)


# minutes, bits: the lengths and depths measured by default (bits None: one depth, and --bits does not apply);
# shapes: for a format of fixed shapes, its table by (minutes, bits), from which --minutes and --bits choose;
# build(directory, minutes, bits) -> [(row fields, path)]; extra(lib, minutes, runs): rows after a case's loads.
Format = collections.namedtuple('Format', 'minutes bits build shapes extra', defaults=(None, None))
FORMATS = {
    'flac': Format((24, 90), (16, 24), build_flac),
    'mkv': Format((24, 90), None, build_mkv, MKV_RATES),
    'truehd': Format((24, 90), (16,), build_truehd),
    'ts': Format((24, 90), (16, 24), build_ts, TS_FILLER),
    'alac': Format((24, 90), (16, 24), build_alac),
    'wavpack': Format((24, 90), (16, 24), build_wavpack),
    'tta': Format((24, 90), (16, 24), build_tta),
    'ps': Format((90,), None, build_ps),
    'ogg': Format((90,), None, build_ogg),
    'mp2': Format((90,), None, build_mp2, extra=ffmpeg_mp2),
    'swr': Format((24, 90), (16,), build_swr, extra=swr_alone),
}


# Every format the tool measures: FORMATS, and the formats added after tests/test_load_tool.py's table of input kinds,
# which tests/test_load_tool_ape.py, tests/test_load_tool_tak.py and tests/test_load_tool_avi.py build in the same way.
ALL_FORMATS = dict(FORMATS, ape=Format((24, 90), (16, 24), build_ape), tak=Format((24, 90), (16, 24), build_tak),
                   avi=Format((90,), (16, 24), build_avi))


def cases(name, minutes, bits):
    """[(minutes, bits)] of one format: its defaults, or those asked for when it can build them."""
    fmt = ALL_FORMATS[name]
    out = [(m, b) for m in minutes or fmt.minutes for b in ([None] if fmt.bits is None else bits or fmt.bits)]
    for m, b in out:
        if m < 1:
            raise ValueError('%s: a length of %d minutes' % (name, m))
        if fmt.bits is not None and b not in fmt.bits:
            raise ValueError('%s is built at %s bits only, not %d' % (name, ' or '.join(map(str, fmt.bits)), b))
        if fmt.shapes is not None and (m, b) not in fmt.shapes:
            raise ValueError('%s has shapes for (minutes, bits) %s only, not %s' % (name, list(fmt.shapes), (m, b)))
    return out


def measure(lib, files, runs):
    """One untimed load of each file, then `runs` rounds of the timed legs in order: one JSON line each."""
    for row, path in files:
        if row['input'] not in LEGS:
            load_once(lib, path, row.get('ffmpeg_audio', False))       # warm-up: page cache, device pool
    for r in range(runs):
        for row, path in files:
            kind = row['input']
            if kind in LEGS:
                out = LEGS[kind](path)
            else:
                wall, phases = load_once(lib, path, row.get('ffmpeg_audio', False))
                out = {'wall_ms': round(1e3 * wall, 1), 'kernel_ms': phases}
                if kind in PROBES:
                    out.update(PROBES[kind](path))
            print(json.dumps(dict(row, run=r, **out)), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('formats', nargs='+', choices=list(ALL_FORMATS), metavar='FORMAT', help=' '.join(ALL_FORMATS))
    ap.add_argument('--minutes', type=int, nargs='+')
    ap.add_argument('--bits', type=int, nargs='+')
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    args = ap.parse_args()
    try:
        plan = [(name, cases(name, args.minutes, args.bits)) for name in args.formats]
    except ValueError as e:
        ap.error(str(e))
    lib = _native.lib()
    lib.sb_profile_enable(1)
    sms = sm_count()
    directory = tempfile.mkdtemp(prefix='load_', dir=args.dir)
    try:
        for name, todo in plan:
            print(json.dumps({'format': name, 'card': card(), 'sms': sms}), flush=True)
            for minutes, bits in todo:
                files = ALL_FORMATS[name].build(directory, minutes, bits)
                measure(lib, files, args.runs)
                if ALL_FORMATS[name].extra:
                    ALL_FORMATS[name].extra(lib, minutes, args.runs)
                for path in {path for _, path in files}:
                    os.remove(path)
            print(json.dumps({'card_after': card()}), flush=True)
    finally:
        shutil.rmtree(directory, ignore_errors=True)


if __name__ == '__main__':
    main()
