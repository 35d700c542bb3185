"""Host-side parts of transcoding and of the decoder's device output, without a device: the release order of
openh264_b200.transcode.OutputOrder driven by a fake decoder, the refused output sizes, and the argument checks of
b2h264_dec_decode_device / b2h264_dec_set_stream."""
import pytest

from openh264_b200.transcode import OutputOrder, Transcoder, check_scale


class FakeDecoder:
    """hands back pictures in decoding order with picture_order()'s values: (poc, flags, reorder depth) per unit"""

    def __init__(self, units):
        self.units = units

    def run(self, q):
        out = []
        for k, (poc, flags, depth) in enumerate(self.units):
            out += q.push(k, poc, flags, depth)
        return out, q.drain()


def test_release_order_without_reordering():
    q = OutputOrder()
    got, rest = FakeDecoder([(0, 1, 0), (2, 0, 0), (4, 0, 0), (0, 1, 0), (2, 0, 0)]).run(q)
    assert got == [0, 1, 2, 3, 4] and rest == []


def test_release_order_b_pyramid_idr_and_flush():
    # I0 P8 B4 b2 b6 | IDR: I0 P4 B2 — decoding order with counts; output by count inside each IDR period, at most 2 held back
    units = [(0, 1, 2), (16, 0, 2), (8, 2, 2), (4, 2, 2), (12, 2, 2), (0, 1, 2), (8, 0, 2), (4, 2, 2)]
    q = OutputOrder()
    got, rest = FakeDecoder(units).run(q)
    assert got + rest == [0, 3, 2, 4, 1, 5, 7, 6]
    assert got == [0, 3, 2, 4, 1, 5] and rest == [7, 6]          # the IDR releases the whole first period; flush the rest


def test_release_order_holds_no_more_than_the_depth():
    q = OutputOrder()
    assert q.push("a", 4, 1, 2) == [] and q.push("b", 2, 0, 2) == []
    assert q.push("c", 6, 0, 2) == ["b"]
    assert q.drain() == ["a", "c"] and q.drain() == []


@pytest.mark.parametrize("dst", [(962, 540), (960, 541), (1920, 1088), (3840, 2160), (8, 8)])
def test_refused_output_sizes(dst):
    with pytest.raises(ValueError):
        check_scale(1920, 1080, *dst)
    with pytest.raises(ValueError):
        Transcoder(1920, 1080, 1, dst_w=dst[0], dst_h=dst[1])       # before any device work


def test_accepted_output_sizes():
    for dst in ((1920, 1080), (960, 540), (640, 360), (1280, 720)):
        check_scale(1920, 1080, *dst)


def test_device_output_entry_points_refuse_null_without_a_device():
    from openh264_b200.binding import load
    L = load()
    assert L.b2h264_dec_decode_device(None, None, None, None, None) == -1
    assert L.b2h264_dec_set_stream(None, None) == -1
