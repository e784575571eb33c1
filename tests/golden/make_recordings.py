#!/usr/bin/env python3
"""Regenerates the real-speech fixtures of the long-form tests (tests/test_long.py) under tests/golden/: four of the
reference project's recordings of spoken digit lists (Matlab/语音样本/, 8 kHz 8-bit mono WAV), copied byte for byte under
ASCII names. Their file names are their transcripts:

  digits_1_10_a.wav       12345678910.wav              "1 2 3 4 5 6 7 8 9 10"
  digits_1_10_b.wav       12345678910 (1).wav          the same list, a second take
  digits_1_9_units_a.wav  123456789十百千万 (1).wav    "1 2 3 4 5 6 7 8 9 十 百 千 万" (10, 100, 1000, 10000)
  digits_1_9_units_b.wav  123456789十百千万 (3).wav    the same list, another take

The machines that run the tests need no checkout of the reference: they read these copies.
Run:  python tests/golden/make_recordings.py REFERENCE_DIR
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
RECORDINGS = {
    "digits_1_10_a.wav": "12345678910.wav",
    "digits_1_10_b.wav": "12345678910 (1).wav",
    "digits_1_9_units_a.wav": "123456789十百千万 (1).wav",
    "digits_1_9_units_b.wav": "123456789十百千万 (3).wav",
}


def main():
    src_dir = os.path.join(sys.argv[1] if len(sys.argv) > 1 else "reference", "Matlab", "语音样本")
    for dst, src in RECORDINGS.items():
        shutil.copyfile(os.path.join(src_dir, src), os.path.join(HERE, dst))
        print("copied", src, "->", dst)


if __name__ == "__main__":
    main()
