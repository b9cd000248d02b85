"""ctypes binding of libsushi_b200.so (the C ABI in include/sushi_b200.h).

There is deliberately no fallback: if the shared library is missing, or no H100 is
visible, every entry point raises.  The CPU implementation of this path lives in
oracle/ and is test infrastructure only.
"""
import ctypes
import os

from .common import SushiError

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libsushi_b200.so')

SB_OK = 0
SB_U8, SB_F32 = 0, 1
ABI_VERSION = 9
SB_TS_PCM_BLURAY, SB_TS_TRUEHD = 0, 1

c_i64 = ctypes.c_int64
c_i64p = ctypes.POINTER(ctypes.c_int64)
c_f32p = ctypes.POINTER(ctypes.c_float)
c_vp = ctypes.c_void_p
c_i32p = ctypes.POINTER(ctypes.c_int32)

# name -> (restype, argtypes); the test-suite checks this table against the header.
PROTOTYPES = {
    'sb_init': (ctypes.c_int, [ctypes.c_int]),
    'sb_shutdown': (ctypes.c_int, []),
    'sb_abi_version': (ctypes.c_int, []),
    'sb_last_error': (ctypes.c_char_p, []),
    'sb_sync': (ctypes.c_int, []),
    'sb_set_block_size': (ctypes.c_int, [ctypes.c_int]),
    'sb_get_block_size': (ctypes.c_int, []),
    'sb_set_engine': (ctypes.c_int, [ctypes.c_int]),
    'sb_set_max_parts': (ctypes.c_int, [c_i64]),
    'sb_get_engine': (ctypes.c_int, []),
    'sb_set_hop_mode': (ctypes.c_int, [ctypes.c_int]),
    'sb_set_premac_mode': (ctypes.c_int, [ctypes.c_int]),
    'sb_set_epilogue': (ctypes.c_int, [ctypes.c_int]),
    'sb_get_epilogue': (ctypes.c_int, []),
    'sb_get_stream': (c_vp, []),
    'sb_pinned_alloc': (ctypes.c_int, [c_i64, ctypes.POINTER(c_vp)]),
    'sb_pinned_free': (ctypes.c_int, [c_vp]),
    'sb_device_alloc': (ctypes.c_int, [c_i64, ctypes.POINTER(c_vp)]),
    'sb_device_free': (ctypes.c_int, [c_vp]),
    'sb_copy_to_host': (ctypes.c_int, [c_vp, c_vp, c_i64]),
    'sb_copy_to_device': (ctypes.c_int, [c_vp, c_vp, c_i64]),
    'sb_copy_on_device': (ctypes.c_int, [c_vp, c_vp, c_i64]),
    'sb_stream_device_ptr': (c_vp, [c_vp]),
    'sb_stream_create': (ctypes.c_int, [c_vp, c_i64, ctypes.c_int, ctypes.POINTER(c_vp)]),
    'sb_stream_create_device': (ctypes.c_int, [c_vp, c_i64, ctypes.c_int, ctypes.POINTER(c_vp)]),
    'sb_stream_destroy': (ctypes.c_int, [c_vp]),
    'sb_stream_length': (c_i64, [c_vp]),
    'sb_stream_dtype': (ctypes.c_int, [c_vp]),
    'sb_stream_read': (ctypes.c_int, [c_vp, c_i64, c_i64, c_vp]),
    'sb_find': (ctypes.c_int, [c_vp, c_vp, c_i64, c_i64, c_i64, c_f32p, c_i64p]),
    'sb_find_batch': (ctypes.c_int, [c_vp, c_vp, c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_f32p, c_i64p]),
    'sb_find_batch_device': (ctypes.c_int, [c_vp, c_vp, c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_vp, c_vp]),
    'sb_match_curves': (ctypes.c_int, [c_vp, c_vp, c_i64, c_i64p, c_i64p, c_i64p, c_i64p, c_f32p]),
    'sb_find_multi': (ctypes.c_int, [ctypes.POINTER(c_vp), ctypes.c_int32, c_i64, c_i32p, c_i32p, c_i64p, c_i64p, c_i64p, c_i64p,
                                     c_f32p, c_i64p]),
    'sb_match_curves_multi': (ctypes.c_int, [ctypes.POINTER(c_vp), ctypes.c_int32, c_i64, c_i32p, c_i32p, c_i64p, c_i64p, c_i64p,
                                             c_i64p, c_f32p]),
    'sb_match_curve': (ctypes.c_int, [c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_f32p]),
    'sb_load_pcm': (ctypes.c_int, [c_vp, c_i64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                   c_i64, c_i64, ctypes.POINTER(c_vp)]),
    'sb_normalise': (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.POINTER(c_vp), c_f32p, c_f32p]),
    'sb_pcm_info': (ctypes.c_int, [c_vp, c_i64p, c_i32p, c_i32p]),
    'sb_pcm_load': (ctypes.c_int, [c_vp, ctypes.c_int, c_i64, c_i64, ctypes.POINTER(c_vp)]),
    'sb_pcm_destroy': (ctypes.c_int, [c_vp]),
    'sb_pcm_from_be': (ctypes.c_int, [c_vp, c_i64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(c_vp)]),
    'sb_flac_decode_file': (ctypes.c_int, [c_vp, c_i64, c_i64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.POINTER(c_vp)]),
    'sb_flac_decode_frames': (ctypes.c_int, [c_vp, c_i64, c_i64p, c_i64p, c_i64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                             ctypes.POINTER(c_vp)]),
    'sb_truehd_decode': (ctypes.c_int, [c_vp, c_i64, c_i64p, c_i64p, c_i64, ctypes.POINTER(c_vp)]),
    'sb_alac_decode_frames': (ctypes.c_int, [c_vp, c_i64, c_i64p, c_i64p, c_i64, c_i32p, ctypes.POINTER(c_vp)]),
    'sb_ts_open': (ctypes.c_int, [ctypes.c_int, ctypes.c_int32, ctypes.c_int32, ctypes.POINTER(c_vp)]),
    'sb_ts_feed': (ctypes.c_int, [c_vp, c_vp, c_i64, c_i64]),
    'sb_ts_finish': (ctypes.c_int, [c_vp, c_i32p, ctypes.POINTER(c_vp)]),
    'sb_ts_destroy': (ctypes.c_int, [c_vp]),
    'sb_comm_unique_id': (ctypes.c_int, [c_vp]),
    'sb_comm_init': (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int]),
    'sb_comm_destroy': (ctypes.c_int, []),
    'sb_comm_world_size': (ctypes.c_int, []),
    'sb_comm_rank': (ctypes.c_int, []),
    'sb_comm_nccl_version': (ctypes.c_int, []),
    'sb_comm_broadcast': (ctypes.c_int, [c_vp, c_i64, ctypes.c_int, ctypes.c_int]),
    'sb_comm_wait': (ctypes.c_int, [ctypes.c_int]),
    'sb_comm_all_gather': (ctypes.c_int, [c_vp, c_vp, c_i64]),
    'sb_comm_max_f32': (ctypes.c_int, [c_f32p, ctypes.c_int]),
    'sb_comm_barrier': (ctypes.c_int, []),
    'sb_timer_start': (ctypes.c_int, []),
    'sb_timer_stop': (ctypes.c_int, [c_f32p]),
    'sb_profile_enable': (ctypes.c_int, [ctypes.c_int]),
    'sb_profile_reset': (ctypes.c_int, []),
    'sb_profile_get': (ctypes.c_int, [ctypes.c_char_p, ctypes.POINTER(ctypes.c_double), c_i64p]),
    'sb_profile_names': (ctypes.c_char_p, []),
    'sb_launch_count': (c_i64, []),
}

_lib = None
_device = None


def load_library():
    """Load the shared library and attach prototypes. No GPU needed for this step."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SushiError(
            'sushi_b200: {0} is missing -- build it with `python -c "import __graft_entry__ as g; g.build()"` '
            '(or `make -C sushi_b200/csrc`). There is no CPU fallback for this path.'.format(LIB_PATH))
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)       # AttributeError here = header/library drift: fail loudly
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.sb_abi_version() != ABI_VERSION:
        raise SushiError('sushi_b200: ABI version mismatch (library {0}, binding {1})'.format(
            lib.sb_abi_version(), ABI_VERSION))
    _lib = lib
    return lib


def check(rc, what=''):
    if rc != SB_OK:
        msg = _lib.sb_last_error().decode('utf-8', 'replace') if _lib is not None else ''
        raise SushiError('sushi_b200 {0} failed (code {1}): {2}'.format(what, rc, msg))


def lib(device=None):
    """The initialised library, bound to one GPU (one process drives one GPU)."""
    global _device
    l = load_library()
    if _device is None:
        if device is None:
            device = int(os.environ.get('SUSHI_B200_DEVICE', os.environ.get('LOCAL_RANK', '0')))
        check(l.sb_init(int(device)), 'sb_init')
        _device = int(device)
    elif device is not None and int(device) != _device:
        raise SushiError('sushi_b200: already bound to GPU {0}, cannot rebind to {1}'.format(_device, device))
    return l


def bound_device():
    return _device


def pinned_empty(shape, dtype):
    """numpy array over page-locked host memory (freed when the array is garbage collected)."""
    import numpy as np
    import weakref
    l = lib()
    dt = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dt.itemsize
    p = c_vp()
    check(l.sb_pinned_alloc(max(nbytes, 1), ctypes.byref(p)), 'sb_pinned_alloc')
    buf = (ctypes.c_uint8 * max(nbytes, 1)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dt, count=int(np.prod(shape))).reshape(shape)
    weakref.finalize(buf, l.sb_pinned_free, p)
    return arr
