"""The encoder's reference state machine (openh264_b200/csrc/enc_refs.h) built without CUDA and played against the receiver scripts
of tests/golden/ltr.json: its per-picture decisions (IDR, frame_num, ref_pic_list_modification, MMCOs, long_term_reference_flag,
max_num_ref_frames, pictures the reference does not code) equal the slice headers and call logs of the reference encoder, and the picture store slots it hands out are
never the reference picture's and stay within the store."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "ltr.json")))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("enc_refs") / "enc_refs_test")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "openh264_b200", "csrc"),
                           os.path.join(ROOT, "tests", "wels", "enc_refs_test.cpp"), "-o", exe])
    return exe


def play(exe, case, tmp):
    cabac, cx, nref, ltr, period, n = case["config"]
    scr = os.path.join(tmp, "script.txt")
    with open(scr, "w") as f:
        f.write("\n".join(case["script"]) + "\n")
    out = subprocess.run([exe, str(nref), str(ltr), str(period), str(n), scr], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    head = lines[0].split()
    pics, failed = [], []
    for ln in lines[1:]:
        t = ln.split()
        if t[2] == "failed":
            failed.append(int(t[1]))
            continue
        idr, fn = int(t[2]), int(t[3])
        k, mods, mmco = 4, [], []
        if t[k] == "mod":
            mods.append([int(t[k + 1]), int(t[k + 2])])
            k += 3
        while t[k] == "mmco":
            op = int(t[k + 1])
            mmco.append([op, int(t[k + 2])] + ([int(t[k + 3])] if op == 3 else []))
            k += 4 if op == 3 else 3
        lt, rec, ref = int(t[k + 1]), int(t[k + 3]), int(t[k + 5])
        pics.append((int(t[1]), [idr, fn, mods, mmco, lt], rec, ref))
    return int(head[1]), int(head[3]), pics, failed


def failed_in(log):
    return [int(ln.split()[1]) for ln in log.splitlines() if " failed " in ln]


@pytest.mark.parametrize("name", sorted(GOLD["cases"]))
def test_decisions_equal_reference_slice_headers(tmp_path, harness, name):
    case = GOLD["cases"][name]
    sps_num_ref, slots, pics, failed = play(harness, case, str(tmp_path))
    assert [p[1] for p in pics] == case["syntax"]
    assert failed == failed_in(case["log"])
    assert set(case["sps_num_ref"]) == {sps_num_ref}
    assert slots == (4 if case["config"][3] else 2)
    for _, syn, rec, ref in pics:
        assert 0 <= rec < slots and rec != ref


def test_dropped_picture_is_covered():
    """the goldens hold a recovery request the reference cannot serve (no confirmed long-term picture): that picture fails"""
    assert any(failed_in(c["log"]) for c in GOLD["cases"].values()) and GOLD["wrap"]["failed"]


def test_frame_num_wrap(tmp_path, harness):
    """32,800 pictures: frame_num wraps at 32,768 amid marks, confirmations, recovery requests and a marking failure; the
    decisions from picture WRAP_FROM on, and the pictures that are dropped, equal the reference's"""
    case = GOLD["wrap"]
    _, _, pics, failed = play(harness, case, str(tmp_path))
    assert [[i] + syn for i, syn, _, _ in pics if i >= case["from"]] == case["syntax"]
    assert failed == case["failed"]
    assert any(s[2] == 0 and not s[1] for s in case["syntax"])          # a P picture with frame_num 0: the wrap
