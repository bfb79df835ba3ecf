"""--mask / --break at the edges of fpl_ext.cu (cases.MASK_BREAK_EDGE_SETS on cases.mask_break_edge_batch) against the oracle:
records, the output-read and mask-region lists, both Stats blocks and the counters; the FASTQ text path (fpl_emit_fastq_host)
and the packed device batch (fpl_emit_batch_device).  That the batch reaches each edge is asserted on the oracle's lists by
tests/test_ext_helpers_host.py:test_edge_batch_reaches_every_edge.  Runs on the GPU and, with FPL_EMULATE=1, on the emulated
library."""
import pytest

import cases
import test_gpu_emit
import test_gpu_emit_batch
import test_gpu_mask_break

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def batch():
    return cases.mask_break_edge_batch()


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_EDGE_SETS))
def test_mask_break_edges(name, batch):
    test_gpu_mask_break.check(cases.MASK_BREAK_EDGE_SETS[name], batch, f"{name}/edges")


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_EDGE_SETS))
def test_mask_break_edges_text(name, batch):
    test_gpu_emit.check(cases.MASK_BREAK_EDGE_SETS[name], batch, f"{name}/edges/text")


@pytest.mark.parametrize("name", sorted(cases.MASK_BREAK_EDGE_SETS))
def test_mask_break_edges_device_batch(name, batch):
    test_gpu_emit_batch.check(cases.MASK_BREAK_EDGE_SETS[name], batch, f"{name}/edges/batch")
