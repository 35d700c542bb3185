"""Host-side parts of the transcoding ladder (openh264_b200.transcode.Transcoder with rungs), without a device: the refused rung
lists, the step-buffer layout and down-sampler descriptor table of a 1080p ladder, and the split of the host entropy threads."""
from fractions import Fraction

import pytest

from openh264_b200 import transcode as T
from openh264_b200.binding import DsPlane

LADDER_1080 = [dict(width=1920, height=1080, qp=26), dict(width=1280, height=720, qp=28), dict(width=960, height=540, qp=30),
               dict(width=640, height=360, qp=32)]


@pytest.fixture
def no_device(monkeypatch):
    """any decoder or encoder the constructor would make fails the test: refusals must come before anything is allocated"""
    def refuse(*a, **k):
        raise AssertionError("allocated before the rungs were checked")
    monkeypatch.setattr(T, "BatchDecoder", refuse)
    monkeypatch.setattr(T, "BatchEncoder", refuse)


@pytest.mark.parametrize("rungs", [
    [dict(width=1920, height=1080), dict(width=2560, height=1440)],     # larger than the source
    [dict(width=1920, height=1088)],                                   # taller than the source
    [dict(width=962, height=540)],                                     # width not divisible by 4
    [dict(width=960, height=541)],                                     # odd height
    [dict(width=1920 - 4 * k, height=1080) for k in range(9)],         # 9 rungs
    [],                                                                # no rungs
    [dict(width=960, height=540, qp=30), dict(width=960, height=540, qp=30)],
    [dict(width=960, height=540), dict(width=960, height=540, qp=26, entropy_threads=3)],   # the same once defaults are filled in
    [dict(width=960, height=540, bitrate=1)],                          # not an encoder keyword
    [dict(width=960)],                                                 # no height
])
def test_refused_rungs(no_device, rungs):
    with pytest.raises(ValueError):
        T.Transcoder(1920, 1080, 2, rungs=rungs)


def test_rungs_and_single_output_arguments_are_exclusive(no_device):
    with pytest.raises(ValueError):
        T.Transcoder(1920, 1080, 2, dst_w=960, dst_h=540, rungs=[dict(width=960, height=540)])
    with pytest.raises(ValueError):
        T.Transcoder(1920, 1080, 2, qp=30, rungs=[dict(width=960, height=540)])


def test_accepted_rungs_differ_in_size_or_configuration():
    got = T.check_rungs(1920, 1080, LADDER_1080 + [dict(width=640, height=360, qp=32, entropy_cabac=True)])
    assert [(w, h) for w, h, _ in got] == [(1920, 1080), (1280, 720), (960, 540), (640, 360), (640, 360)]
    assert got[4][2] == dict(qp=32, entropy_cabac=True)


def _ratio(src, dst, scale):
    return int(Fraction(src, dst) * scale + Fraction(1, 2))


def test_descriptor_table_of_the_1080p_ladder():
    offsets, pitch, planes = T.ladder_layout(1920, 1080, [(r["width"], r["height"]) for r in LADDER_1080])
    # the decoded picture is the 1080p rung (offset 0); every other size follows at a 256-byte aligned offset
    sizes = [1920 * 1080 * 3 // 2, 1280 * 720 * 3 // 2, 960 * 540 * 3 // 2, 640 * 360 * 3 // 2]
    aligned = [-(-b // 256) * 256 for b in sizes]
    assert aligned == [3110400, 1382400, 777728, 345600]
    starts = [sum(aligned[:k]) for k in range(4)]
    assert offsets == {(1920, 1080): starts[0], (1280, 720): starts[1], (960, 540): starts[2], (640, 360): starts[3]}
    assert pitch == sum(aligned) == 5616128
    # Y, U, V of 1280x720 (general ratio: 3 luma, 4 chroma), 960x540 (half: 0), 640x360 (one third: 2)
    want, row = [], 0
    src_off = [0, 1920 * 1080, 1920 * 1080 + 960 * 540]
    for (w, h), start, (mode_y, mode_c) in zip([(1280, 720), (960, 540), (640, 360)], starts[1:], [(3, 4), (0, 0), (2, 2)]):
        dst_off = [0, w * h, w * h + (w // 2) * (h // 2)]
        for pl in range(3):
            c = 1 if pl else 0
            sw, sh, dw, dh = 1920 >> c, 1080 >> c, w >> c, h >> c
            mode = mode_c if c else mode_y
            sx = _ratio(sw, dw, 1 << (16 if mode == 3 else 15)) if mode >= 3 else 0
            sy = _ratio(sh, dh, 1 << 15) if mode >= 3 else 0
            want.append((mode, sx, sy, sw, sh, sw, dw, dh, dw, row, src_off[pl], start + dst_off[pl]))
            row += dh
    assert planes == want
    assert [p[9] for p in planes] == [0, 720, 1080, 1440, 1980, 2250, 2520, 2880, 3060]
    assert (planes[0][1], planes[0][2], planes[1][1], planes[1][2]) == (98304, 49152, 49152, 49152)
    assert [f for f, _ in DsPlane._fields_] == ["mode", "sx", "sy", "src_w", "src_h", "src_stride", "dst_w", "dst_h", "dst_stride",
                                                "row0", "src_offset", "dst_offset"]


def test_layout_without_a_source_size_rung_and_shared_sizes():
    # no rung at the source size: the decoded picture lives elsewhere, the first rung is at offset 0; two rungs of one size
    # (different encoder settings) read one down-scaled picture
    offsets, pitch, planes = T.ladder_layout(1920, 1080, [(960, 540), (640, 360), (960, 540)])
    assert offsets == {(960, 540): 0, (640, 360): 777728}
    assert pitch == 777728 + 345600 and len(planes) == 6


def test_layout_puts_the_source_size_first_whatever_its_rung():
    # the decoder writes the decoded picture at offset 0 of the row: a source-size rung given after others must sit there
    for sizes in ([(960, 540), (1920, 1080)], [(1280, 720), (640, 360), (1920, 1080), (640, 360)]):
        offsets, pitch, planes = T.ladder_layout(1920, 1080, sizes)
        assert offsets[(1920, 1080)] == 0
        assert sorted(offsets.values())[1] == 3110400 and min(p[11] for p in planes) == 3110400
        assert pitch == 3110400 + sum(-(-(w * h * 3 // 2) // 256) * 256 for w, h in set(sizes) - {(1920, 1080)})
    offsets, _, planes = T.ladder_layout(1920, 1080, [(960, 540), (1920, 1080)])
    assert offsets == {(1920, 1080): 0, (960, 540): 3110400}
    assert [p[11] for p in planes] == [3110400, 3110400 + 960 * 540, 3110400 + 960 * 540 + 480 * 270]
    assert T.ladder_layout(1920, 1080, [(1920, 1080), (960, 540)]) == T.ladder_layout(1920, 1080, [(960, 540), (1920, 1080)])


def test_single_output_layout_is_one_picture_per_row():
    for dst in ((1920, 1080), (960, 540), (1280, 720)):
        offsets, pitch, planes = T.ladder_layout(1920, 1080, [dst])
        assert offsets == {dst: 0} and pitch == (dst[0] * dst[1] * 3 // 2 + 255) & ~255
        assert len(planes) == (0 if dst == (1920, 1080) else 3)


@pytest.mark.parametrize("cores", [1, 2, 3, 4, 8, 13, 64])
def test_entropy_thread_split(cores):
    mbs = [8160, 3600, 2040, 920]                                      # 1080p, 720p, 540p, 360p
    n = T.entropy_threads(mbs, cores)
    assert min(n) >= 1
    assert sum(n) == max(cores, len(mbs)) if cores >= len(mbs) else all(x == 1 for x in n)
    assert n == sorted(n, reverse=True)                                # more macroblocks, no fewer threads
    assert T.entropy_threads([8160], cores) == [cores]
