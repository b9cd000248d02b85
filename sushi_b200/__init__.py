"""sushi_b200 -- H100-native implementation of tp7/Sushi's audio template-matching path.

Public surface (mirrors the reference's wav.py / the part of sushi.py that drives it):
    WavStream            drop-in stream class, GPU-backed find_substream
    SushiError, clip     as in the reference's common.py
    calculate_shifts     the shift solver (sushi.py:400-508) batched onto the GPU matcher
    calculate_shifts_many, shift_events_many, shift_scripts, find_substreams
                         many episodes at once: every ready search of every episode in one launch
    prepare_search_groups, groups_from_chapters, ...   the grouping heuristics (sushi.py:67-216,309-397)
"""
from .common import SushiError, clip, format_time   # noqa: F401
from .wavstream import WavStream, DownmixedWavFile, find_substreams   # noqa: F401
from .events import ScriptEvent   # noqa: F401
from .shifts import calculate_shifts, calculate_shifts_many   # noqa: F401
from .grouping import (prepare_search_groups, merge_short_lines_into_groups, groups_from_chapters,   # noqa: F401
                       split_broken_groups, fix_near_borders, smooth_events, detect_groups, average_shifts,
                       interpolate_nones, running_median)

__version__ = '0.1.0'
from .script import AssScript, SrtScript, AssEvent, SrtEvent, load_script   # noqa: F401,E402
from .pipeline import shift_events, shift_events_many, shift_script, shift_scripts   # noqa: F401,E402
