"""Generates tests/golden/merge_golden.json from the UNMODIFIED reference binary (run where oracle/_ref/fastplong_ref has been
built by `make -C oracle`): for every run of tests/test_gpu_merge.py's MERGE_RUNS and every worker count T of its THREADS, the
md5 of the masked -h report (tests/html_golden.py:mask) and of the -j report without its "command" line, of `fastplong_ref -w T`,
with the md5 of the input FASTQ they were made from.

Usage:  python tests/golden/make_golden_merge.py
"""
import hashlib
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
import report_twin  # noqa: E402
import test_gpu_merge as tm  # noqa: E402
from oracle_lib import RefEngine  # noqa: E402


def main():
    out = {}
    for name in tm.MERGE_RUNS:
        opt, batch = html_golden.run_input(name)
        e = RefEngine(opt)                 # the reference's own operators: its lists, for the empty-read counts
        res = e.process(batch)
        pre, post = report_html_twin.read_lists(batch.lens, res, e.segments() if tm.is_ext(opt) else None)
        empty = html_golden.empties(pre, post)
        g = {"input_md5": html_golden.input_md5(batch), "html_md5": {}, "json_md5": {}}
        for T in tm.THREADS:
            with tempfile.TemporaryDirectory() as d:
                html, js = tm.run_reference(name, T, d)
            g["html_md5"][str(T)] = html_golden.masked_md5(html, empty)
            g["json_md5"][str(T)] = hashlib.md5(report_twin.without_command(js)).hexdigest()
        out[name] = g
        print(name, g)
    json.dump(out, open(tm.FIXTURE, "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
