"""Long-term references and loss-recovery feedback through layer 3 (ISVCEncoder): one driver binary
(tests/wels/wels_ltr_driver.cpp, compiled against the reference's public headers staged under oracle/_ref/include) plays the
receiver scripts of tests/golden/ltr.json against openh264_b200/libopenh264_b200_wels.so; bitstream and call log equal what the
unmodified reference produced, and the compiled reference is run beside it where it is present."""
import hashlib
import json
import os

import pytest

import ltr_cases as L

GOLD = json.load(open(os.path.join(L.ROOT, "tests", "golden", "ltr.json")))
need_api = pytest.mark.skipif(not os.path.isdir(L.API_INC), reason="the reference's public headers (oracle/_ref/include) are not present")
need_ours = pytest.mark.skipif(not os.path.exists(L.OURLIB), reason="layer 3 is built where the reference headers exist (build())")


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return L.build_driver(str(tmp_path_factory.mktemp("ltr_driver")))


def case_tuple(name):
    c = GOLD["cases"][name]
    return tuple(c["config"]) + (c["script"],), c


@pytest.mark.gpu
@need_api
@need_ours
@pytest.mark.parametrize("name", sorted(GOLD["cases"]))
def test_drop_in_with_ltr(tmp_path, driver, name):
    case, gold = case_tuple(name)
    r, bs, log = L.run(driver, L.OURLIB, case, gold["script"], str(tmp_path), "b2")
    assert r.returncode == 0, r.stderr
    assert log == gold["log"]
    assert L.ref_syntax(bs) == gold["syntax"]
    assert hashlib.sha1(bs).hexdigest() == gold["sha1"]
    if os.path.exists(L.REFLIB):
        r2, bs2, log2 = L.run(driver, L.REFLIB, case, gold["script"], str(tmp_path), "ref")
        assert r2.returncode == 0 and bs2 == bs and log2 == log


def test_goldens_use_committed_clip():
    """the clip the goldens were made from is the committed one"""
    assert hashlib.sha1(open(L.CLIP, "rb").read()).hexdigest() == GOLD["clip_sha1"]


@pytest.mark.gpu
@need_api
@need_ours
def test_ltr_option_on_running_stream(tmp_path, driver):
    """ENCODER_OPTION_LTR on a running stream: asking for the setting the stream has is accepted and changes nothing; switching
    LTR off is refused (it would move the stream to another pool) and the stream carries on as before"""
    case, gold = case_tuple("ltr_p30_cavlc_high")
    script = sorted(gold["script"] + ["3 ltropt 1", "5 ltropt 0"], key=lambda s: int(s.split()[0]))
    r, bs, log = L.run(driver, L.OURLIB, case, script, str(tmp_path), "opt")
    assert r.returncode == 0, r.stderr
    assert "3 ltropt 1 -> 0" in log
    assert "5 ltropt 0 -> 0" not in log and "5 ltropt 0 -> " in log
    assert hashlib.sha1(bs).hexdigest() == gold["sha1"]
