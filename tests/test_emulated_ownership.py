"""Who owns the library's device memory, streams and events, on the emulated library (tests/simt_emu.py), whose cudaMalloc /
cudaMallocHost count the blocks alive (emu_live_allocs) and fail the k-th allocation from now on request (emu_fail_alloc), and whose
stream and event creations do the same (emu_live_handles, emu_fail_handle) and count the calls that get a handle that is not live
(emu_bad_handles).  A context frees everything its entry points allocated or created when it is destroyed; an allocation that fails
anywhere in a call makes the call fail and leaks nothing; so does a stream or event creation, except a timing event, whose launch
then runs untimed; fpl_stats_reserve is all or nothing; a report or emit build that failed gives the same bytes when it is called
again.  Whether a call succeeds or fails, fpl_launch_count goes up by the kernels it ran, as the emulator counts them
(emu_launches)."""
import dataclasses
import gc

import numpy as np
import pytest

import cases
import layouts
import simt_emu
from fastplong_b200 import abi, pack, synth
from fastplong_b200.binding import FplError

PLAIN, EXT = cases.OPTION_SETS["cut_polyx_cplx"], cases.MASK_BREAK_SETS["mask_and_break"]
BATCH = cases.blocky_quality_batch(5, n=12)
TEXT = b"".join(b"@r%d\n%s\n+\n%s\n" % (i, *BATCH.read(i)) for i in range(BATCH.n_reads))
EMPTY = pack.PackedBatch(*(np.zeros(pack.TAIL_PAD, np.uint8) for _ in range(2)), np.zeros(3, np.int64), np.zeros(3, np.int32))
# every base Q2: with --mask/--break no output read is left, so no post-filter segment
VANISH = dataclasses.replace(BATCH, qual=np.full_like(BATCH.qual, ord("#")))
# kernels outside fpl_launch_count: fpl_process_device's length reduction, the --mask/--break stage, the FASTQ ingest, and
# fpl_eval_adapter_kmers (no context's); cub's and NCCL's kernels are not emulator launches
UNCOUNTED = (b"k_lens_minmax", b"k_ext_", b"k_count_lines", b"k_fastq_", b"k_eval_")


@pytest.fixture(scope="module")
def lib():
    return simt_emu.emulated_library()


def engine(opt):
    e = simt_emu.EmuEngine(opt)
    e.keep_read_lists()
    return e


def process_device(e, batch):
    """fpl_process_device on copies of the batch that the engine keeps (device memory is host memory here)"""
    size = abi.batch_bytes(batch.n_bytes)
    e.dev = [np.zeros(size, np.uint8), np.zeros(size, np.uint8), batch.offsets.astype(np.int64), batch.lens.astype(np.int32)]
    e.dev[0][:batch.n_bytes], e.dev[1][:batch.n_bytes] = batch.seq, batch.qual
    e.process_device(*(a.ctypes.data for a in e.dev), batch.n_reads, batch.n_bytes)


def emit_batch(e):
    return [bytes(t.numpy()) for b in e.emit_batch(True, device="cpu") for t in (b.seq, b.qual, b.offsets, b.lens, b.segs)]


def with_source(e):
    """e and e.src, another context with the same options, have processed a batch: fpl_merge_stats(e, [e.src]) is ready"""
    e.process(BATCH)
    e.src = engine(e.options)
    e.src.process(BATCH)


def with_image(e):
    """e has processed a batch, e.image is the state of another context that has: fpl_state_merge(e, [e.image]) is ready"""
    e.process(BATCH)
    src = engine(e.options)
    src.process(BATCH)
    e.image = src.export_state()
    src.close()


def counted(lib, e, call):
    """call(e), which may raise; either way fpl_launch_count has gone up by the counted kernels the emulator ran"""
    def ran():
        return lib.emu_launches(b"") - sum(lib.emu_launches(p) for p in UNCOUNTED)
    before = e.launch_count, ran()
    try:
        return call(e)
    finally:
        assert e.launch_count - before[0] == ran() - before[1], "fpl_launch_count against the kernels run"


def close(e):
    for x in (e, getattr(e, "src", None)):
        if x:
            x.close()


# entry point -> (what the context has done before, the call); the calls marked True are retried after a failure
ENTRIES = {
    "fpl_process_host": (None, lambda e: e.process(BATCH), False),
    "fpl_process_device": (None, lambda e: process_device(e, BATCH), False),
    "fpl_process_fastq_host": (None, lambda e: e.process_fastq(TEXT), False),
    "fpl_emit_fastq_host": (lambda e: e.process_fastq(TEXT), lambda e: e.emit_fastq(True), True),
    "fpl_emit_batch_device": (lambda e: e.process(BATCH), emit_batch, True),
    "fpl_report_json": (lambda e: e.process(BATCH), lambda e: e.report_json(command="fastplong -i x"), True),
    "fpl_report_html": (lambda e: e.process(BATCH), lambda e: e.report_html(command="fastplong -i x", time_text="t"), True),
    "fpl_merge_stats": (with_source, lambda e: e.merge(e.src), False),
    "fpl_stats_reserve": (lambda e: e.process(BATCH), lambda e: e.reserve_cycles(1 << 14), False),
    "fpl_state_merge": (with_image, lambda e: e.merge_state(e.image), False),
    "fpl_process_host of empty reads": (None, lambda e: e.process(EMPTY), False),
    "fpl_process_host of reads without output": (None, lambda e: e.process(VANISH), False),
    "fpl_report_json on a fresh context": (lambda e: None, lambda e: e.report_json(command="fastplong -i x"), True),
}


def live(lib):
    gc.collect()
    return lib.emu_live_allocs()


@pytest.mark.parametrize("opt", [PLAIN, EXT], ids=["plain", "mask_break"])
def test_a_context_frees_everything_it_allocated(lib, opt):
    base = live(lib)
    e = engine(opt)
    e.process(BATCH)
    e.emit_batch(True, device="cpu")
    process_device(e, BATCH)
    e.emit_batch(True, device="cpu")
    e.process_fastq(TEXT)
    e.emit_fastq(True)
    e.emit_batch(True, device="cpu")
    e.report_json()
    e.report_html(time_text="t")
    src = engine(opt)
    src.process(BATCH)
    e.merge(src)
    e.report_html(time_text="t")
    e.reset()
    e.process(synth.ont_like(4, 3000, 11))      # longer than the first capacity: the Stats blocks grow
    e.close()
    src.close()
    assert live(lib) == base


@pytest.mark.parametrize("opt", [PLAIN, EXT], ids=["plain", "mask_break"])
def test_a_failed_fpl_create_leaks_nothing(lib, opt):
    base, k = live(lib), 0
    while True:
        k += 1
        lib.emu_fail_alloc(k)
        try:
            engine(opt).close()
            failed = False
        except FplError:
            failed = True
        pending = lib.emu_fail_alloc(0)
        assert live(lib) == base, f"allocation {k} failed: leak"
        if pending:
            assert not failed and k > 1
            return
        assert failed, f"allocation {k} failed, fpl_create succeeded"


@pytest.mark.parametrize("entry", list(ENTRIES))
@pytest.mark.parametrize("opt", [PLAIN, EXT], ids=["plain", "mask_break"])
def test_an_allocation_failure_leaks_nothing(lib, opt, entry):
    """every allocation the call makes fails once in turn: the call fails and leaks nothing; a report or emit call made again
    gives what a context that never failed gives"""
    before, call, retry = ENTRIES[entry]
    want = None
    if retry:
        e = engine(opt)
        before(e)
        want = call(e)
        close(e)
    base, k = live(lib), 0
    while True:
        k += 1
        e = engine(opt)
        if before:
            before(e)
        lib.emu_fail_alloc(k)
        try:
            counted(lib, e, call)
            failed = False
        except FplError:
            failed = True
        pending = lib.emu_fail_alloc(0)
        if pending:
            assert not failed and k > 1, f"{entry} allocates nothing here"
        else:
            assert failed, f"{entry}: allocation {k} failed, the call succeeded"
            if retry:
                assert counted(lib, e, call) == want, f"{entry} retried after allocation {k} failed"
        close(e)
        assert live(lib) == base, f"{entry}: allocation {k} failed: leak"
        if pending:
            return


def test_a_failed_fpl_stats_reserve_changes_nothing(lib):
    e, fresh = engine(PLAIN), engine(PLAIN)
    for x in (e, fresh):
        x.process(BATCH)
    cycles, stats = e.cycles, [e.stats(w) for w in (0, 1)]
    lib.emu_fail_alloc(2)                    # the second of the two new blocks
    with pytest.raises(FplError):
        e.reserve_cycles(4 * cycles)
    assert lib.emu_fail_alloc(0) == 0
    assert e.cycles == cycles
    for w in (0, 1):
        np.testing.assert_array_equal(e.stats(w), stats[w])
    longer = synth.ont_like(4, 3000, 11)      # longer than the capacity: the blocks grow and take the rows along
    for x in (e, fresh):
        x.process(longer)
    assert e.cycles == fresh.cycles > cycles
    for w in (0, 1):
        np.testing.assert_array_equal(e.stats(w), fresh.stats(w))
    np.testing.assert_array_equal(e.counters(), fresh.counters())
    e.close()
    fresh.close()


# ENTRIES, fpl_reset, and fpl_process_host on three reads whose slots lie 1 MiB apart: at FPL_PIECE_MB=1 it uploads them on its
# copy stream in three pieces, an event each
PIECES = layouts.relayout(BATCH.slice(0, 3), align=1 << 20)
HANDLE_ENTRIES = {**ENTRIES, "fpl_process_host in pieces": (None, lambda e: e.process(PIECES), False),
                  "fpl_reset": (lambda e: e.process(BATCH), lambda e: e.reset(), False)}


def held(lib):
    """live blocks, live streams and events, calls that got a handle that was not live"""
    return live(lib), lib.emu_live_handles(), lib.emu_bad_handles()


@pytest.mark.parametrize("timing", [False, True], ids=["untimed", "timed"])
@pytest.mark.parametrize("opt", [PLAIN, EXT], ids=["plain", "mask_break"])
def test_every_entry_point_releases_its_streams_events_and_blocks(lib, monkeypatch, opt, timing):
    monkeypatch.setenv("FPL_PIECE_MB", "1")
    base = held(lib)
    for entry, (before, call, _) in HANDLE_ENTRIES.items():
        e = engine(opt)
        e.set_timing(timing)
        if before:
            before(e)
        counted(lib, e, call)
        close(e)
        assert held(lib) == base, entry


def test_a_failed_stream_creation_in_fpl_create_leaks_nothing(lib):
    base, k = held(lib), 0
    while True:
        k += 1
        lib.emu_fail_handle(k)
        try:
            engine(PLAIN).close()
            failed = False
        except FplError:
            failed = True
        pending, kind = lib.emu_fail_handle(0), lib.emu_failed_handle_kind()
        assert held(lib) == base, f"creation {k} failed: leak or dead handle"
        if pending:
            assert not failed and k > 1
            return
        assert failed and kind == simt_emu.EMU_STREAM, f"creation {k} failed, fpl_create succeeded"


@pytest.mark.parametrize("timing", [False, True], ids=["untimed", "timed"])
@pytest.mark.parametrize("entry", list(HANDLE_ENTRIES))
@pytest.mark.parametrize("opt", [PLAIN, EXT], ids=["plain", "mask_break"])
def test_a_failed_stream_or_event_creation_leaks_nothing(lib, monkeypatch, opt, entry, timing):
    """every stream or event the call creates fails once in turn: the call fails, except where a timing event failed, whose launch
    then runs untimed and is counted; nothing leaks, no call gets a poisoned or released handle, and the context's next batch gives
    the records, Stats and counters of a context that never failed"""
    monkeypatch.setenv("FPL_PIECE_MB", "1")
    before, call, _ = HANDLE_ENTRIES[entry]

    def run(k, skip=False):
        """-> (the call failed, what the k-th creation made (0: it never came), timed launches, launches, the next batch's
        records, Stats and counters); skip: the call is left out"""
        e = engine(opt)
        e.set_timing(timing)
        if before:
            before(e)
        lib.emu_fail_handle(k)
        failed = False
        try:
            if not skip:
                counted(lib, e, call)
        except FplError:
            failed = True
        kind = lib.emu_failed_handle_kind() if lib.emu_fail_handle(0) == 0 else 0
        timed = sum(n for _, n in e.kernel_times().values())
        launches = e.launch_count
        res = e.process(BATCH)
        after = [res.tobytes(), *(e.stats(w).tobytes() for w in (0, 1)), e.counters().tobytes()]
        close(e)
        return failed, kind, timed, launches, after

    _, _, timed, launches, after = run(0)
    after_skip = run(0, skip=True)[4]
    base, k = held(lib), 0
    while True:
        k += 1
        failed, kind, got_timed, got_launches, got_after = run(k)
        assert held(lib) == base, f"{entry}: creation {k} failed: leak or dead handle"
        if not kind:
            return
        if kind == simt_emu.EMU_TIMING_EVENT:
            assert not failed, f"{entry}: timing event {k} failed, so did the call"
            assert (got_timed, got_launches) == (timed - 1, launches), f"{entry}: timing event {k} failed: timed launches, launches"
            assert got_after == after, f"{entry}: the batch after timing event {k} failed"
        else:
            assert failed, f"{entry}: creation {k} failed, the call succeeded"
            assert got_after == after_skip, f"{entry}: the batch after creation {k} failed"
