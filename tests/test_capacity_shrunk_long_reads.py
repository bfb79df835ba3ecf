"""Long reads of every segment-decision shape on the emulated library built with the shrunk constants of
tests/test_capacity_shrunk.py (RQ_LONG 300, RQ_LIST 2, one SM): the cases tests/test_gpu_long_read_decisions.py runs at
the product's sizes — split long reads on k_read_qual's block-wide list and past it (the fast scan), the same reads through
k_read_qual_exc (the jit scan), dropped reads beside them, the --mask/--break path — against the oracle, in the CPU suite."""
import test_gpu_long_read_decisions as rq
from test_capacity_shrunk import SCANS, engine, shrunk

BUILD = "group_of_2_stages"


def test_long_read_decisions_shrunk():
    lib, k = shrunk(BUILD)
    rq.run_cases(lambda opt, scan: engine(BUILD, opt, scan), SCANS, k, BUILD)
