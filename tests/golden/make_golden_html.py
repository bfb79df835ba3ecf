"""Generates tests/golden/html_golden.json from the UNMODIFIED reference binary (run where oracle/_ref/fastplong_ref has been
built by `make -C oracle`): for every run of tests/html_golden.py, the md5 of the input FASTQ, how many reads of each Stats
block have no bases (the quirk-1 tail the mask drops), and the md5 of the masked -h report of `fastplong_ref -w 1`.

Usage:  python tests/golden/make_golden_html.py
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import html_golden  # noqa: E402
import report_html_twin  # noqa: E402
from oracle_lib import REF_BIN, RefEngine  # noqa: E402


def main():
    out = {}
    for name in html_golden.RUNS:
        opt, batch = html_golden.run_input(name)
        e = RefEngine(opt)                 # the reference's own operators: its lists, for the empty-read counts
        res = e.process(batch)
        ext = opt.to_abi()[0].mask_enabled or opt.to_abi()[0].break_enabled
        pre, post = report_html_twin.read_lists(batch.lens, res, e.segments() if ext else None)
        empty = html_golden.empties(pre, post)
        with tempfile.TemporaryDirectory() as d:
            text = html_golden.run_reference(REF_BIN, name, d)
        out[name] = {"input_md5": html_golden.input_md5(batch), "empty": empty, "html_md5": html_golden.masked_md5(text, empty),
                     "bytes": len(text)}
        print(name, out[name])
    json.dump(out, open(html_golden.FIXTURE, "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
