"""Generates tests/golden/slices.json from the UNMODIFIED reference (oracle/_ref, built by oracle/Makefile.ref): for every case of
tests/slices_cases.py, the SHA-1 of the clip and of the reference encoder's bitstream, and its call log (whether InitializeExt
accepted the configuration, the slice argument GetOption reports resolved, and the NAL sizes of every layer of every picture).

It also checks the claim that makes the multi-threaded cases bit-exact: fixed slices coded by 4 threads without load balancing
give the bytes of one thread with loop filter idc 2, which the reference codes whenever more than one thread codes slices.

    python tests/golden/make_slices_golden.py"""
import hashlib
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import slices_cases as S  # noqa: E402


def main():
    tmp = tempfile.mkdtemp()
    exe = S.build_driver(tmp)
    gold = {"clips": {}, "cases": {}, "refused_both": {}}
    for name in S.CLIPS:
        gold["clips"][name] = hashlib.sha1(S.clip(name).tobytes()).hexdigest()
    for name, c in S.CASES.items():
        r, bs, log = S.run_case(exe, S.REFLIB, name, tmp)
        assert r.returncode == 0 and "accepted" in log, (name, r.stderr, log)
        gold["cases"][name] = {"sha1": hashlib.sha1(bs).hexdigest(), "log": log}
        print(name, len(bs), "bytes", log.splitlines()[1])
    # 4 threads without load balancing: the bytes of one thread, loop filter idc 0 coded as 2
    c = S.CASES["fixed4_threads4_cavlc_low"]
    w, h, n = S.CLIPS[c[0]]
    one = S.run(exe, S.REFLIB, S.clip(c[0]), w, h, n, c[1], c[2], c[3], c[4], (2,) + c[5][1:], c[6], (1, 0), tmp, "one_thread")
    assert one[1] == open(os.path.join(tmp, "fixed4_threads4_cavlc_low.264"), "rb").read(), "4 threads differ from 1 thread"
    for name, (w, h, slices, threads) in S.REFUSED_BOTH.items():
        yuv = S.clip("synth_96x64")[:0]
        r, _, log = S.run(exe, S.REFLIB, yuv, w, h, 1, 28, (0, 66), S.HIGH, 0, (0, 0, 0), slices, threads, tmp, name)
        assert r.returncode == 0 and "refused" in log, (name, log)
        gold["refused_both"][name] = log
    for name, (w, h, slices, threads) in S.REFUSED_OURS.items():
        yuv = S.clip("CiscoVT2people_320x192")
        r, _, log = S.run(exe, S.REFLIB, yuv, w, h, 1, 28, (0, 66), S.HIGH, 0, (0, 0, 0), slices, threads, tmp, name)
        assert r.returncode == 0 and "accepted" in log, (name, log)
    with open(os.path.join(HERE, "slices.json"), "w") as f:
        json.dump(gold, f, indent=1)


if __name__ == "__main__":
    main()
