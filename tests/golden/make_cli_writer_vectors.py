"""Copies the txt / srt / vtt files the reference's command line wrote next to its `.words.json` results into
tests/golden/subtitles/ (build container only; the copies are committed because /root/reference does not exist on the
GPU box): tests/expected/punctuations_{yes,no}/{punctuations.mp3,bonjour.wav}.{txt,srt,vtt,words.srt,words.vtt}.
The `.words.json` inputs are copied by make_subtitles_vectors.py.  These are data fixtures of the reference's
test-suite, not source code; tests/test_cli_writers.py replays them.
"""
import os
import shutil

REF = "/root/reference/tests/expected"
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "subtitles")


def main():
    n = 0
    for folder in ("punctuations_yes", "punctuations_no"):
        for stem in ("punctuations.mp3", "bonjour.wav"):
            for ext in ("txt", "srt", "vtt", "words.srt", "words.vtt"):
                dst = f"{HERE}/{folder}_{stem}.{ext}"
                shutil.copyfile(f"{REF}/{folder}/{stem}.{ext}", dst)
                os.chmod(dst, 0o644)
                n += 1
    print(n, "files")


if __name__ == "__main__":
    main()
