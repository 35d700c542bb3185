"""Writes tests/golden/intra_mb.json: SHA-1s of what the UNMODIFIED reference decides and codes on the intra macroblock cases
of tests/intra_mb_cases.py (oracle/_ref, ref_shim.cpp:ref_intra_mb: WelsMdI16x16 then WelsMdIntraSecondaryModesEnc), one per
(content class, QP) group of the compared fields (intra_mb_cases.fields), plus the case count and one SHA-1 of the
reference's (I16x16, I4x4, chroma) costs.  The cost limits of the limit cases come from the reference's own run without one.
    python tests/golden/make_intra_mb_golden.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import h264lib  # noqa: E402
import intra_mb_cases as ic  # noqa: E402


def main():
    assert h264lib.have_ref(), "oracle/_ref is not built"
    base, kinds, qps = ic.base_cases()
    cases, kinds, qps = ic.with_limits(base, kinds, qps, lambda c: ic.run_ref(c)[0])
    out, costs = ic.run_ref(cases)
    golden = {"cases": int(len(cases)), "costs": h264lib.sha1(costs), "groups": ic.group_hashes(out, kinds, qps)}
    with open(os.path.join(HERE, "intra_mb.json"), "w") as f:
        json.dump(golden, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(cases)} cases, {len(golden['groups'])} groups")


if __name__ == "__main__":
    main()
