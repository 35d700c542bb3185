"""The batching core shared by the broker's encoder and decoder pools (openh264_b200/wels/batcher.h), without a GPU:
tests/wels/batcher_test.cpp puts a fake coder behind it that records each batch.  The program is built twice, plainly and
with ThreadSanitizer, and each case must run clean in both builds:
  many     T threads x P calls on one pool: every call returns its own slot's result, no batch holds a slot twice or a slot
           that is not pending, T x P pictures are coded in all;
  fail     every caller of a failed batch gets the failure, the callers of the next batch succeed;
  lone     a lone registered slot does not wait for the window (B2H264_BROKER_WAIT_US = 10 s);
  release  a release issued during a batch returns only after the batch's step has returned, and resets the stream."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WELS = os.path.join(ROOT, "openh264_b200", "wels")
FLAGS = {"plain": ["-O2"], "tsan": ["-O1", "-fsanitize=thread"]}


@pytest.fixture(scope="module", params=sorted(FLAGS))
def program(request, tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("batcher") / "batcher_test")
    r = subprocess.run(["g++", "-std=c++17", "-g", "-Wall", "-pthread"] + FLAGS[request.param] +
                       ["-I", WELS, os.path.join(ROOT, "tests", "wels", "batcher_test.cpp"), os.path.join(WELS, "batcher.cpp"), "-o", exe],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "warning" not in r.stderr, r.stderr
    return exe


@pytest.mark.parametrize("case", ["many", "fail", "lone", "release"])
def test_batcher(program, case):
    r = subprocess.run([program, case], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stdout + r.stderr
    assert case + ": ok" in r.stdout
