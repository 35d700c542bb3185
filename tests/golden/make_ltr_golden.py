"""Generates tests/golden/ltr.json from the UNMODIFIED reference (oracle/_ref, built by oracle/Makefile.ref): for every case of
tests/ltr_cases.py, the script the receiver played, the SHA-1 of the reference encoder's bitstream, its call log, the reference
syntax of every picture's slice header, max_num_ref_frames of its SPS, and the SHA-1 of every picture the reference decoder
decodes from it.

The script of an LTR case is the fixed receiver calls of the case plus marking feedback found by playing the receiver against
the reference: every picture the encoder marks long-term (an IDR with long_term_reference_flag, or a P picture with MMCOs) is
confirmed two pictures later.  Each new confirmation changes what the encoder marks next, so the reference is run again until
the script stops changing.  A recovery request that comes while no long-term picture is confirmed makes the reference's
EncodeFrame fail for that picture; the log records it ("frame N failed 2") and the next picture is an IDR.

The "wrap" entry is a long case for the CPU test of the reference state machine only: 32,800 pictures, so that frame_num wraps
at 32,768, with marks, confirmations, recovery requests and a marking failure around the wrap.  It stores the syntax of the
pictures from WRAP_FROM on and the pictures that failed.

    python tests/golden/make_ltr_golden.py"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ltr_cases as L  # noqa: E402


def confirmations(syntax, pictures, fixed):
    """marking-success feedback two pictures after every marked picture (pictures: the picture index of each coded picture)"""
    taken = {int(s.split()[0]) for s in fixed if " mf " in s}
    out = []
    for i, (idr, fn, _, mmco, lt) in zip(pictures, syntax):
        if (idr and lt) or mmco:
            at = i + 2
            if at < pictures[-1] and at not in taken:
                out.append(f"{at} mf 4 cur {fn}")
    return out


def decoded_sha1s(bs, tmp):
    src, out = os.path.join(tmp, "dec.264"), os.path.join(tmp, "dec.yuv")
    with open(src, "wb") as f:
        f.write(bs)
    subprocess.run([L.REFDEC, src, out], capture_output=True, timeout=300)
    data = open(out, "rb").read()
    fsz = L.W * L.H * 3 // 2
    return [hashlib.sha1(data[k:k + fsz]).hexdigest() for k in range(0, len(data), fsz)]


def main():
    tmp = tempfile.mkdtemp()
    exe = L.build_driver(tmp)
    gold = {"clip": os.path.basename(L.CLIP), "clip_sha1": hashlib.sha1(open(L.CLIP, "rb").read()).hexdigest(),
            "width": L.W, "height": L.H, "qp": L.QP, "cases": {}}
    for name, case in L.CASES.items():
        fixed = list(case[6])
        script = list(fixed)
        for _ in range(40):
            r, bs, log = L.run(exe, L.REFLIB, case, script, tmp, name)
            assert r.returncode == 0, r.stderr
            if not case[3]:
                break
            nxt = sorted(set(fixed) | set(confirmations(L.ref_syntax(bs), L.coded_pictures(log), fixed)),
                         key=lambda s: int(s.split()[0]))
            if nxt == script:
                break
            script = nxt
        syn = L.ref_syntax(bs)
        gold["cases"][name] = {"config": list(case[:6]), "script": script, "sha1": hashlib.sha1(bs).hexdigest(), "log": log,
                               "syntax": syn, "sps_num_ref": L.sps_num_ref(bs), "decoded_sha1": decoded_sha1s(bs, tmp)}
        print(name, len(bs), "bytes", log.count(" failed "), "dropped,", sum(1 for s in syn if s[0]), "IDR", sum(1 for s in syn if s[2] and s[2][0][0] == 2), "LTR refs")
    case = L.WRAP
    r, bs, log = L.run(exe, L.REFLIB, case, case[6], tmp, "wrap")
    assert r.returncode == 0, r.stderr
    pics = L.coded_pictures(log)
    syn = L.ref_syntax(bs)
    gold["wrap"] = {"config": list(case[:6]), "script": case[6], "from": L.WRAP_FROM,
                    "syntax": [[i] + s for i, s in zip(pics, syn) if i >= L.WRAP_FROM],
                    "failed": [int(ln.split()[1]) for ln in log.splitlines() if " failed " in ln]}
    print("wrap", len(gold["wrap"]["syntax"]), "pictures kept,", gold["wrap"]["failed"], "failed")
    with open(os.path.join(HERE, "ltr.json"), "w") as f:
        json.dump(gold, f, indent=1)


if __name__ == "__main__":
    main()
