"""Regenerates tests/golden/cli_sample_xz.json: the information lines (tests/test_zz_reference_cli.py:info_lines) the
reference's UNMODIFIED command-line program prints on support/sample.xz when it is linked against the UNMODIFIED
reference library oracle/_ref/libnrsc5_ref.so - for the whole capture from a file and from stdin, and for its first
20 MB.  Needs oracle/_ref/ built where the reference tree is; the JSON is committed.

    python tests/golden/make_golden_cli.py
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "cli"), os.path.join(ROOT, "oracle")]

import build_cli  # noqa: E402
import common  # noqa: E402
import reftap  # noqa: E402
import test_zz_reference_cli as t  # noqa: E402


def main():
    ctl = build_cli.build(reftap.REF_SO, "ref")
    raw = common.load_sample().tobytes()
    out = {"source": "the reference CLI (src/main.c, src/log.c) linked against the unmodified reference library, "
                     "`nrsc5 -r <file or -> -o out.wav 0` on support/sample.xz",
           "input_fnv": common.fnv1a32(raw[:1 << 20])}
    with tempfile.TemporaryDirectory() as td:
        full, part = os.path.join(td, "sample"), os.path.join(td, "sample20")
        open(full, "wb").write(raw)
        open(part, "wb").write(raw[:t.PREFIX_BYTES])
        out["prefix_20mb"] = t.info_lines(t.run_cli(ctl, part, td))
        out["full_file"] = t.info_lines(t.run_cli(ctl, full, td))
        out["full_stdin"] = t.info_lines(t.run_cli(ctl, full, td, stdin=True))
    json.dump(out, open(os.path.join(HERE, "cli_sample_xz.json"), "w"), indent=0)
    print({k: len(v) for k, v in out.items() if isinstance(v, list)})


if __name__ == "__main__":
    main()
