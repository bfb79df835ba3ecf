"""The fused k_cycle_stats pass on the emulated library built with the shrunk constants of tests/test_capacity_shrunk.py
(CS_STAGE 24, CS_GROUP 48 and 60): post starts on both sides of CS_REACH, split reads, post lists past CS_STAGE and
CS_GROUP, and the packed counter and both 16-bit 5-mer halves at their fullest — the cases tests/test_gpu_fused_post.py
runs at the product's sizes — against the oracle, in the CPU suite."""
import pytest

import capacity
import test_gpu_fused_post as fused
from test_capacity_shrunk import BUILDS, engine, shrunk


@pytest.mark.parametrize("build", sorted(BUILDS))
def test_post_starts(build):
    for s in fused.STARTS:
        opt = fused.trim_opt(s)
        capacity.compare_with_oracle(engine(build, opt), opt, fused.start_batch(s, 100 + s), f"{build}/start{s}")


@pytest.mark.parametrize("build", sorted(BUILDS))
def test_post_lists_and_headroom(build):
    lib, k = shrunk(build)
    opt = fused.trim_opt(5)
    for count in capacity.cycle_counts(k):
        capacity.compare_with_oracle(engine(build, opt), opt, fused.post_list_batch(k, count), f"{build}/post_list{count}")
    for base in "AC":
        capacity.compare_with_oracle(engine(build, fused.HEADROOM_OPT), fused.HEADROOM_OPT, fused.headroom_batch(k, base),
                                     f"{build}/headroom/{base}")
