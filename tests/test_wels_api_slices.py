"""SM_FIXEDSLCNUM_SLICE and SM_RASTER_SLICE through layer 3.  One driver binary (tests/wels/wels_slices_driver.cpp, compiled here
against the reference's public headers staged under oracle/_ref/include) runs the compiled reference and our library side by
side: the same bitstream, the same call log (one NAL per slice, in the reference's layer layout), the same slice argument
reported by GetOption, and the same refusal where the reference refuses.  Where the reference's bytes would depend on the
machine (fixed slices with load balancing, an automatic slice or thread count) or on the bits spent (SM_SIZELIMITED_SLICE),
InitializeExt refuses."""
import json
import os

import pytest

import h264lib
import slices_cases as S

GOLD = json.load(open(os.path.join(h264lib.ROOT, "tests", "golden", "slices.json")))
need_ref = pytest.mark.skipif(not (os.path.isdir(S.API_INC) and os.path.exists(S.REFLIB)),
                              reason="the reference build (library and public headers) is not present")
need_ours = pytest.mark.skipif(not os.path.exists(S.OURLIB), reason="layer 3 is built where the reference headers exist (build())")


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return S.build_driver(str(tmp_path_factory.mktemp("slices_driver")))


@need_ref
def test_reference_matches_golden(tmp_path, driver):
    """the committed hashes are the reference's own output"""
    import hashlib
    for name in ["rows_cavlc_high", "fixed4_threads4_cavlc_low", "small_runs_single"]:
        r, bs, log = S.run_case(driver, S.REFLIB, name, str(tmp_path))
        assert r.returncode == 0, r.stderr
        assert hashlib.sha1(bs).hexdigest() == GOLD["cases"][name]["sha1"] and log == GOLD["cases"][name]["log"]


@pytest.mark.gpu
@need_ref
@need_ours
@pytest.mark.parametrize("name", sorted(S.CASES))
def test_drop_in_with_slices(tmp_path, driver, name):
    import hashlib
    r, bs, log = S.run_case(driver, S.OURLIB, name, str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert hashlib.sha1(bs).hexdigest() == GOLD["cases"][name]["sha1"]
    assert log == GOLD["cases"][name]["log"]


@pytest.mark.gpu
@need_ref
@need_ours
@pytest.mark.parametrize("name", sorted(S.REFUSED_BOTH) + sorted(S.REFUSED_OURS))
def test_drop_in_refusals(tmp_path, driver, name):
    w, h, slices, threads = {**S.REFUSED_BOTH, **S.REFUSED_OURS}[name]
    yuv = S.clip("CiscoVT2people_320x192")
    r, _, log = S.run(driver, S.OURLIB, yuv, w, h, 1, 28, (0, 66), S.HIGH, 0, (0, 0, 0), slices, threads, str(tmp_path), name)
    assert r.returncode == 0 and log == "InitializeExt refused\n", r.stderr
    assert "unsupported encoder configuration" in r.stderr
    if name in S.REFUSED_BOTH:
        assert GOLD["refused_both"][name] == log
