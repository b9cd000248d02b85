"""ALAC (Apple Lossless) tracks of MP4 / QuickTime and Matroska files: the ALACSpecificConfig the container carries
(an MP4 `alac` box's body, a Matroska A_ALAC track's CodecPrivate) and the call that decodes the frames on the GPU."""
import struct

import numpy as np

from . import _native


def bit_depth(config):
    """The bit depth of an ALACSpecificConfig."""
    return struct.unpack('>IBB', config[:6])[2]


def track_decoder(config):
    """decode(device, table) of an ALAC track (sb_alac_decode_frames on its FrameTable).  `config` is the 24-byte
    ALACSpecificConfig: frame length, bit depth, pb, mb, kb, channels and sample rate reach the decoder."""
    fl, _, depth, pb, mb, kb, channels, _, _, _, rate = struct.unpack('>IBBBBBBHIII', config[:24])
    cfg = np.array([fl, depth, pb, mb, kb, channels, rate], np.int32)
    return lambda device, table: _native.decode_frames(device, 'sb_alac_decode_frames', table.data, table.offset,
                                                       table.block, cfg.ctypes.data_as(_native.c_i32p))
