"""Timecodes, keyframe and chapter files (sushi_b200.timing), and the closest-keyframe distance:
ports of the reference's tests/timecodes.py (without get_frame_number, which nothing on this path
uses), tests/main.py:168-181 and tests/demuxing.py:130-173, plus keyframe-file cases."""
import pytest

from sushi_b200.common import SushiError
from sushi_b200.grouping import get_distance_to_closest_kf
from sushi_b200.timing import (Timecodes, load_keyframe_times, parse_keyframes, parse_ogm_start_times,
                               parse_scxvid_keyframes, parse_xml_start_times)

VFR_V1 = '# timecode format v1\nAssume 23.976000\n0,2000,29.970000\n3000,4000,59.940000'


# tests/timecodes.py: CfrTimecodesTestCase
def test_cfr_get_frame_time_zero():
    assert Timecodes.cfr(23.976).get_frame_time(0) == 0


def test_cfr_get_frame_time_sane():
    assert Timecodes.cfr(23.976).get_frame_time(10) == pytest.approx(10.0 / 23.976, abs=1e-7)


def test_cfr_get_frame_time_insane():
    assert Timecodes.cfr(23.976).get_frame_time(100000) == pytest.approx(100000.0 / 23.976, abs=1e-7)


def test_cfr_get_frame_size():
    tcs = Timecodes.cfr(23.976)
    t1, t2 = tcs.get_frame_size(0), tcs.get_frame_size(1000)
    assert t1 == pytest.approx(1.0 / 23.976, abs=1e-7)
    assert t1 == pytest.approx(t2, abs=1e-7)


# tests/timecodes.py: TimecodesTestCase
def test_cfr_timecodes_v2():
    parsed = Timecodes.parse('# timecode format v2\n' + '\n'.join(str(1000 * x / 23.976) for x in range(0, 30000)))
    assert parsed.get_frame_size(0) == pytest.approx(1.0 / 23.976, abs=1e-7)
    assert parsed.get_frame_size(25) == pytest.approx(1.0 / 23.976, abs=1e-7)
    assert parsed.get_frame_time(100) == pytest.approx(1.0 / 23.976 * 100, abs=1e-7)
    assert parsed.get_frame_time(0) == 0


def test_cfr_timecodes_v1():
    parsed = Timecodes.parse('# timecode format v1\nAssume 23.976024')
    assert parsed.get_frame_size(0) == pytest.approx(1.0 / 23.976024, abs=1e-7)
    assert parsed.get_frame_size(25) == pytest.approx(1.0 / 23.976024, abs=1e-7)
    assert parsed.get_frame_time(100) == pytest.approx(1.0 / 23.976024 * 100, abs=1e-7)
    assert parsed.get_frame_time(0) == 0


def test_cfr_timecodes_v1_with_overrides():
    parsed = Timecodes.parse('# timecode format v1\nAssume 23.976000\n0,2000,23.976000\n3000,5000,23.976000')
    assert parsed.get_frame_size(0) == pytest.approx(1.0 / 23.976, abs=1e-7)
    assert parsed.get_frame_size(25) == pytest.approx(1.0 / 23.976, abs=1e-7)
    assert parsed.get_frame_time(100) == pytest.approx(1.0 / 23.976 * 100, abs=1e-7)
    assert parsed.get_frame_time(0) == 0


def test_vfr_timecodes_v1_frame_size_at_first_frame():
    assert Timecodes.parse(VFR_V1).get_frame_size(timestamp=0) == pytest.approx(1.0 / 29.97, abs=1e-7)


def test_vfr_timecodes_v1_frame_size_outside_of_defined_range():
    assert Timecodes.parse(VFR_V1).get_frame_size(timestamp=5000.0) == pytest.approx(1.0 / 23.976, abs=1e-7)


def test_vfr_timecodes_v1_frame_size_inside_override_block():
    assert Timecodes.parse(VFR_V1).get_frame_size(timestamp=49.983) == pytest.approx(1.0 / 29.97, abs=1e-7)


def test_vfr_timecodes_v1_frame_size_between_override_blocks():
    assert Timecodes.parse(VFR_V1).get_frame_size(timestamp=87.496) == pytest.approx(1.0 / 23.976, abs=1e-7)


def test_vfr_timecodes_v1_frame_time_at_first_frame():
    assert Timecodes.parse(VFR_V1).get_frame_time(number=0) == pytest.approx(0, abs=1e-7)


def test_vfr_timecodes_v1_frame_time_outside_of_defined_range():
    assert Timecodes.parse(VFR_V1).get_frame_time(number=25000) == pytest.approx(1000.968, abs=5e-4)


def test_vfr_timecodes_v1_frame_time_inside_override_block():
    assert Timecodes.parse(VFR_V1).get_frame_time(number=1500) == pytest.approx(50.05, abs=5e-4)


def test_vfr_timecodes_v1_frame_time_between_override_blocks():
    assert Timecodes.parse(VFR_V1).get_frame_time(number=2500) == pytest.approx(87.579, abs=5e-4)


# fallbacks and errors
def test_v2_without_default_rate_ends_with_frames_of_size_zero():
    parsed = Timecodes.parse('# timestamp format v2\n0\n40\n80\n')
    assert parsed.get_frame_time(10) == 0.08                  # past the end: the last frame's time
    assert parsed.get_frame_size(0.04) == pytest.approx(0.04)
    assert parsed.get_frame_size(0.08) == 0
    assert parsed.get_frame_size(5.0) == 0


def test_v1_without_overrides_is_a_constant_rate():
    parsed = Timecodes.parse('# timecode format v1\nAssume 25')
    assert parsed.times == [] and parsed.get_frame_time(50) == 2.0 and parsed.get_frame_size(7.0) == 0.04


def test_v1_past_the_overrides_continues_at_the_default_rate():
    parsed = Timecodes.parse('# timecode format v1\nAssume 25\n0,9,50')
    assert len(parsed.times) == 11 and parsed.get_frame_time(10) == pytest.approx(0.2)
    assert parsed.get_frame_time(12) == pytest.approx(0.2 + 2 * 0.04)


@pytest.mark.parametrize('text', ['', '# timecode format v3\n0\n', 'garbage'])
def test_unsupported_or_empty_timecodes_are_an_error(text):
    with pytest.raises(SushiError):
        Timecodes.parse(text)


# tests/main.py: GetDistanceToClosestKeyframeTestCase
KEYTIMES = [0, 10, 20, 30, 40, 50, 60, 70, 80, 90, 100]


def test_finds_correct_distance_to_first_keyframe():
    assert get_distance_to_closest_kf(0, KEYTIMES) == 0


def test_finds_correct_distance_to_last_keyframe():
    assert get_distance_to_closest_kf(105, KEYTIMES) == -5


def test_finds_correct_distance_to_keyframe_before():
    assert get_distance_to_closest_kf(63, KEYTIMES) == -3


def test_finds_distance_to_keyframe_after():
    assert get_distance_to_closest_kf(36, KEYTIMES) == 4


def test_distance_tie_goes_to_the_keyframe_before():
    assert get_distance_to_closest_kf(35, KEYTIMES) == -5


# tests/demuxing.py: ExternalChaptersTestCase
def test_parse_xml_start_times():
    text = """<?xml version="1.0"?>
<!-- <!DOCTYPE Chapters SYSTEM "matroskachapters.dtd"> -->
<Chapters>
  <EditionEntry>
    <EditionUID>2092209815</EditionUID>
    <ChapterAtom>
      <ChapterUID>3122448259</ChapterUID>
      <ChapterTimeStart>00:00:00.000000000</ChapterTimeStart>
      <ChapterDisplay>
        <ChapterString>Prologue</ChapterString>
      </ChapterDisplay>
    </ChapterAtom>
    <ChapterAtom>
      <ChapterUID>998777246</ChapterUID>
      <ChapterTimeStart>00:00:17.017000000</ChapterTimeStart>
      <ChapterDisplay>
        <ChapterString>Opening Song ("YES!")</ChapterString>
      </ChapterDisplay>
    </ChapterAtom>
    <ChapterAtom>
      <ChapterUID>55571857</ChapterUID>
      <ChapterTimeStart>00:01:47.023000000</ChapterTimeStart>
      <ChapterDisplay>
        <ChapterString>Part A (Tale of the Doggypus)</ChapterString>
      </ChapterDisplay>
    </ChapterAtom>
  </EditionEntry>
</Chapters>
"""
    assert parse_xml_start_times(text) == [0, 17.017, 107.023]


def test_parse_ogm_start_times():
    text = """CHAPTER01=00:00:00.000
CHAPTER01NAME=Prologue
CHAPTER02=00:00:17.017
CHAPTER02NAME=Opening Song ("YES!")
CHAPTER03=00:01:47.023
CHAPTER03NAME=Part A (Tale of the Doggypus)
"""
    assert parse_ogm_start_times(text) == [0, 17.017, 107.023]


def test_chapters_are_sorted_and_start_at_zero():
    assert parse_ogm_start_times('chapter02=00:01:00.500\nCHAPTER01=00:00:10.000\n') == [0, 10.0, 60.5]


# keyframe files
SCXVID = ('# XviD 2pass stat file (core version 1.1.2)\n# Please do not modify this file\n\n'
          'i 1 0 0 0 0 0 0\np 1 0 0 0 0 0 0\np 1 0 0 0 0 0 0\ni 1 0 0 0 0 0 0\nb 1 0 0 0 0 0 0\ni 1 0 0 0 0 0 0\n')


def test_scxvid_keyframes_are_the_i_lines():
    assert parse_scxvid_keyframes(SCXVID) == [0, 3, 5]


def test_parse_keyframes_file(tmp_path):
    p = tmp_path / 'kf.txt'
    p.write_text(SCXVID)
    assert parse_keyframes(str(p)) == [0, 3, 5]


def test_missing_frame_zero_is_inserted(tmp_path):
    p = tmp_path / 'kf.txt'
    p.write_text(SCXVID.replace('\ni 1', '\np 1', 1))
    assert parse_keyframes(str(p)) == [0, 3, 5]
    p.write_text(SCXVID.replace('i 1', 'p 1'))
    assert parse_keyframes(str(p)) == [0]


def test_unsupported_keyframes_file(tmp_path):
    p = tmp_path / 'kf.txt'
    p.write_text('# keyframe format v1\nfps 0\n0\n24\n')
    with pytest.raises(SushiError, match='Unsupported keyframes type'):
        parse_keyframes(str(p))


def test_load_keyframe_times(tmp_path):
    (tmp_path / 'src.txt').write_text(SCXVID)
    (tmp_path / 'dst.txt').write_text(SCXVID)
    (tmp_path / 'tc.txt').write_text('# timecode format v2\n0\n50\n100\n150\n200\n250\n')
    kt = load_keyframe_times(str(tmp_path / 'src.txt'), str(tmp_path / 'dst.txt'), src_fps=25.0,
                             dst_timecodes=str(tmp_path / 'tc.txt'))
    assert kt.src_keytimes == [0.0, 0.12, 0.2] and kt.dst_keytimes == [0.0, 0.15, 0.25]
    assert kt.src_timecodes.get_frame_size(3.0) == 0.04 and kt.dst_timecodes.get_frame_size(0.1) == pytest.approx(0.05)
