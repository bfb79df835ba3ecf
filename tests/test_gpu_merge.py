"""fpl_merge_stats / Engine.merge: several contexts of one process merged on the device, as SingleEndProcessor::process merges
its workers (Stats::merge, FilterResult::merge in thread order):
  - one batch split over 1, 2, 3 and 5 contexts and merged, into a fresh context and into the first: the words of both Stats
    blocks and of the counters, the JSON and the HTML report equal one context's over the whole batch (and the HTML the twin);
  - the reference binary at -w T: 16-read packs dealt to T contexts as its readerTask deals them, merged in thread order, give
    its -h report (masked) and its -j report (minus the command line), against fresh runs where oracle/_ref/fastplong_ref is
    built and against the md5s of tests/golden/merge_golden.json everywhere;
  - capacities (a source longer than dst, a dst reserved far above, curves past 300 cycles), identities (sources unchanged,
    a source twice, an empty source, no source, processing after the merge), stream ordering, capture, refusals, launches."""
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import cases
import html_golden
import report_html_twin
import report_twin
from fastplong_b200 import Options, pack_reads, synth
from fastplong_b200.binding import Engine, FplError
from oracle_lib import REF_BIN, OracleEngine

pytestmark = pytest.mark.gpu

EMULATED = os.environ.get("FPL_EMULATE", "") not in ("", "0")
TIME = html_golden.TIME
HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "merge_golden.json")
PACK_SIZE = 16                     # src/common.h:33


def deal_packs(reads, T):
    """SingleEndProcessor::readerTask (src/seprocessor.cpp:331-385): pack p, reads [16p, 16p + 16), goes to worker p mod T; each
    worker's reads in the order it receives them"""
    out = [[] for _ in range(T)]
    for p in range(0, (len(reads) + PACK_SIZE - 1) // PACK_SIZE):
        out[p % T] += reads[p * PACK_SIZE:(p + 1) * PACK_SIZE]
    return out


def reads_of(batch):
    return [batch.read(i) for i in range(batch.n_reads)]


def is_ext(opt):
    o = opt.to_abi()[0]
    return bool(o.mask_enabled or o.break_enabled)


def engine(opt, keep=True):
    e = Engine(opt)
    e.keep_read_lists(keep)
    return e


def twin_lists(opt, batches):
    """the (length, median) lists Stats::statRead builds over the batches in order, from the oracle's records"""
    o, pre, post = OracleEngine(opt), [], []
    for b in batches:
        res = o.process(b)
        p, q = report_html_twin.read_lists(b.lens, res, o.segments() if is_ext(opt) else None)
        pre += p
        post += q
    return pre, post


def assert_same(got, want, what="report"):
    if got != want:
        i = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        raise AssertionError(f"{what}s differ at byte {i} of {len(got)} / {len(want)}:\n"
                             f"got:  {got[max(0, i - 160):i + 60]!r}\nwant: {want[max(0, i - 160):i + 60]!r}")


def words(e, W):
    return [e.stats(0, W), e.stats(1, W), e.counters()]


def assert_equal_contexts(got, want, is_rna=False, html=True):
    """both Stats blocks and the counters word for word, the JSON and (html) the HTML report byte for byte"""
    W = max(got.cycles, want.cycles)
    for k, (a, b) in enumerate(zip(words(got, W), words(want, W))):
        np.testing.assert_array_equal(a, b, err_msg=("stats(0)", "stats(1)", "counters")[k])
    assert_same(got.report_json(is_rna=is_rna), want.report_json(is_rna=is_rna), "JSON report")
    if html:
        text = got.report_html(time_text=TIME, is_rna=is_rna)
        assert_same(text, want.report_html(time_text=TIME, is_rna=is_rna), "HTML report")
        return text


def twin_html(e, opt, lists, is_rna=False, **kw):
    return report_html_twin.report(e.stats(0), e.stats(1), e.counters(), opt, lists[0], lists[1], time_text=TIME, is_rna=is_rna, **kw)


# ---- 1. one batch in shards ----
SHARD_SETS = {"default_se": cases.OPTION_SETS["default_se"], "cut_polyx_cplx": cases.OPTION_SETS["cut_polyx_cplx"],
              "fasta64_polyx": cases.OPTION_SETS["fasta64_polyx"], **cases.MASK_BREAK_SETS,
              "rna_adapters": cases.RNA_SETS["rna_adapters"]}


def shard_batch(name):
    if name == "fasta64_polyx":
        return cases.hifi_fasta64_batch(401, n=80, mean=1500)
    if name == "rna_adapters":
        return cases.rna_batch(402, n=80)
    if name in cases.MASK_BREAK_SETS:
        return cases.blocky_quality_batch(403 + len(name), n=80)
    return synth.ont_like(80, 1500, 404 + len(name), p_chimera=0.08, p_polya=0.08, q_mean=17.0)


@pytest.mark.parametrize("name", sorted(SHARD_SETS))
def test_shards_merge_into_one_context(name):
    opt, batch, rna = SHARD_SETS[name], shard_batch(name), name.startswith("rna")
    whole = engine(opt)
    whole.process(batch)
    assert_same(whole.report_html(time_text=TIME, is_rna=rna), twin_html(whole, opt, twin_lists(opt, [batch]), rna), "HTML report")
    reads = reads_of(batch)
    for K in (1, 2, 3, 5):
        cut = np.linspace(0, len(reads), K + 1).astype(int)
        parts = [pack_reads(reads[a:b]) for a, b in zip(cut[:-1], cut[1:])]
        shards = [engine(opt) for _ in range(K)]
        for s, p in zip(shards, parts):
            s.process(p)
        fresh = engine(opt)
        fresh.merge(*shards)
        assert_equal_contexts(fresh, whole, rna)
        shards[0].merge(*shards[1:])
        assert_equal_contexts(shards[0], whole, rna)


# ---- 2. the reference binary at -w T ----
MERGE_RUNS = ("default", "mask_break", "rna", "fasta64")
THREADS = (2, 3, 8)


def run_reference(name, T, workdir):
    """the reference binary at -w T on the run's input: (-h bytes, -j bytes)"""
    opt, batch = html_golden.run_input(name)
    fq = os.path.join(workdir, "in.fq")
    open(fq, "wb").write(html_golden.fastq(batch))
    extra = []
    if opt.adapter_fasta:
        fa = os.path.join(workdir, "adapters.fa")
        with open(fa, "w") as f:        # headers chosen so that std::map order == list order (src/options.cpp:50-59)
            for i, s in enumerate(opt.adapter_fasta):
                f.write(f">a{i:03d}\n{s}\n")
        extra += ["-a", fa]
    html, js = os.path.join(workdir, "r.html"), os.path.join(workdir, "r.json")
    cmd = [REF_BIN, "-i", fq, "-o", os.path.join(workdir, "out.fq"), "-j", js, "-h", html, "-w", str(T)]
    r = subprocess.run(cmd + opt.cli_flags() + extra, capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-2000:])
    return open(html, "rb").read(), open(js, "rb").read()


def merged_workers(name, T):
    """T contexts fed as the reference's workers are, merged in thread order into worker 0: (its HTML, its JSON, the empty-read
    counts the mask drops)"""
    opt, batch = html_golden.run_input(name)
    rna = name in html_golden.IS_RNA
    workers = [engine(opt) for _ in range(T)]
    for w, rs in zip(workers, deal_packs(reads_of(batch), T)):
        if rs:
            w.process(pack_reads(rs))
    workers[0].merge(*workers[1:])
    empty = html_golden.empties(*twin_lists(opt, [batch]))
    html = workers[0].report_html(command="fastplong -i in.fq", title=html_golden.TITLE.get(name, "fastplong report"),
                                  time_text=TIME, is_rna=rna)
    return html, workers[0].report_json(is_rna=rna), empty


def md5(b):
    return hashlib.md5(b).hexdigest()


@pytest.mark.parametrize("T", THREADS)
@pytest.mark.parametrize("name", MERGE_RUNS)
def test_merged_workers_match_reference_threads(name, T, tmp_path):
    _, batch = html_golden.run_input(name)
    assert batch.n_reads % (PACK_SIZE * T), "the last pack must be partial"
    html, js, empty = merged_workers(name, T)
    g = json.load(open(FIXTURE)).get(name, {})
    checked = False
    if g.get("input_md5") == html_golden.input_md5(batch):
        assert html_golden.masked_md5(html, empty) == g["html_md5"][str(T)]
        assert md5(report_twin.without_command(js)) == g["json_md5"][str(T)]
        checked = True
    if os.path.exists(REF_BIN):
        ref_html, ref_js = run_reference(name, T, str(tmp_path))
        assert_same(html_golden.mask(html, empty), html_golden.mask(ref_html, empty), "masked HTML report")
        assert_same(report_twin.without_command(js), report_twin.without_command(ref_js), "JSON report")
        checked = True
    if not checked:
        pytest.skip("no reference binary, and numpy made another input than when the fixture was made")


# ---- 3. capacities ----
def long_reads(seed, lengths):
    rng = np.random.default_rng(seed)
    return [(synth.BASES[rng.integers(0, 4, L)].tobytes(), (rng.integers(3, 45, L).astype(np.uint8) + 33).tobytes()) for L in lengths]


def test_source_longer_than_dst_grows_dst():
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    short, long = pack_reads(long_reads(1, [120, 300, 250] * 5)), pack_reads(long_reads(2, [350, 2000, 7777, 5000] * 3))
    dst, src, whole = engine(opt), engine(opt), engine(opt)
    dst.process(short)
    src.process(long)
    assert src.cycles > dst.cycles
    dst.merge(src)
    assert dst.cycles >= src.cycles
    whole.process(short)
    whole.process(long)
    text = assert_equal_contexts(dst, whole)
    assert b",type:'log'" in text          # the curves past 300 cycles are down-sampled
    assert_same(text, twin_html(dst, opt, twin_lists(opt, [short, long])))


def test_dst_reserved_far_above_the_sources():
    opt = cases.OPTION_SETS["default_se"]
    a, b = synth.ont_like(40, 1500, 11), synth.ont_like(40, 900, 12)
    dst, src, whole = engine(opt), engine(opt), engine(opt)
    dst.reserve_cycles(1 << 16)
    dst.process(a)
    src.process(b)
    dst.merge(src)
    assert dst.cycles == 1 << 16
    whole.process(a)
    whole.process(b)
    assert_equal_contexts(dst, whole)


# ---- 4. identities ----
def snapshot(e):
    return [*words(e, e.cycles), e.report_json(), e.report_html(time_text=TIME)]


def test_sources_unchanged_and_source_twice():
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    b = synth.ont_like(50, 1500, 21, p_chimera=0.1)
    src = engine(opt)
    src.process(b)
    before = snapshot(src)
    dst = engine(opt)
    dst.merge(src, src)
    after = snapshot(src)
    for x, y in zip(before, after):
        np.testing.assert_array_equal(np.frombuffer(x, np.uint8) if isinstance(x, bytes) else x,
                                      np.frombuffer(y, np.uint8) if isinstance(y, bytes) else y)
    W = max(dst.cycles, src.cycles)
    for d, s in zip(words(dst, W), words(src, W)):
        np.testing.assert_array_equal(d, 2 * s)
    pre, post = twin_lists(opt, [b])
    assert_same(dst.report_html(time_text=TIME), twin_html(dst, opt, (pre + pre, post + post)))


def test_empty_and_no_source_change_nothing():
    opt = cases.OPTION_SETS["fasta64_polyx"]
    dst = engine(opt)
    dst.process(cases.hifi_fasta64_batch(22, n=40, mean=1200))
    before = snapshot(dst)
    dst.set_timing(True)
    launches = dst.launch_count
    dst.merge()
    assert dst.launch_count == launches and dst.kernel_times()["k_merge_stats"][1] == 0
    dst.merge(engine(opt))
    assert dst.launch_count == launches + 1
    for x, y in zip(before, snapshot(dst)):
        assert (x == y) if isinstance(x, bytes) else np.array_equal(x, y)


def test_processing_after_the_merge_continues_the_sequence():
    opt = cases.MASK_BREAK_SETS["mask_and_break"]
    b1, b2, b3 = (cases.blocky_quality_batch(30 + k, n=40) for k in range(3))
    dst, src, whole = engine(opt), engine(opt), engine(opt)
    dst.process(b1)
    src.process(b2)
    dst.merge(src)
    dst.process(b3)
    for b in (b1, b2, b3):
        whole.process(b)
    text = assert_equal_contexts(dst, whole)
    assert_same(text, twin_html(dst, opt, twin_lists(opt, [b1, b2, b3])))


# ---- 5. ordering ----
def test_sources_reset_reused_and_destroyed_right_after_the_merge():
    opt = cases.OPTION_SETS["default_se"]
    a, b, c = synth.ont_like(60, 2000, 41), synth.ont_like(60, 2000, 42), synth.ont_like(300, 3000, 43)
    dst, s1, s2, whole = engine(opt), engine(opt), engine(opt), engine(opt)
    s1.process(a)
    s2.process(b)
    dst.merge(s1, s2)
    s1.reset()                            # no sync in between: stream-ordered behind the merge
    s1.process(c)
    s2.close()
    whole.process(a)
    whole.process(b)
    assert_equal_contexts(dst, whole)


# ---- 6. capture and refusals ----
def test_source_without_capture_refuses_html_keeps_json():
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    a, b = synth.ont_like(40, 1500, 51), synth.ont_like(40, 1500, 52)
    dst, src, whole = engine(opt), engine(opt, keep=False), engine(opt)
    dst.process(a)
    src.process(b)
    dst.merge(src)
    with pytest.raises(FplError, match="capture"):
        dst.report_html(time_text=TIME)
    whole.process(a)
    whole.process(b)
    assert_equal_contexts(dst, whole, html=False)
    off = engine(opt, keep=False)          # a destination with capture off copies no list: incomplete
    off.merge(engine(opt))
    with pytest.raises(FplError, match="capture"):
        off.report_html(time_text=TIME)


def test_refusals_leave_dst_unchanged():
    opt = cases.OPTION_SETS["fasta5"]
    dst, src = engine(opt), engine(opt)
    b = pack_reads(cases.planted_fasta_reads(61, n=40))
    dst.process(b)
    src.process(b)
    before = words(dst, dst.cycles)
    lib = dst.lib

    def refused(srcs, n=None, d=dst.h, match=""):
        arr = (C.c_void_p * max(1, len(srcs)))(*srcs)
        assert lib.fpl_merge_stats(d, arr, len(srcs) if n is None else n) < 0
        msg = lib.fpl_last_error().decode()
        assert match in msg, msg

    refused([src.h.value], d=None, match="null destination")
    refused([src.h.value, None], match="source 1 is null")
    refused([src.h.value], n=-1, match="negative")
    refused([src.h.value, dst.h.value], match="source 1 is the destination")
    fa = cases.OPTION_SETS["fasta5"].adapter_fasta
    kw = dict(start_adapter=synth.ADAPTER_START, adapter_fasta=fa, trim_poly_x=True, poly_x_min_len=8)
    for change, why in ((dict(poly_x_min_len=9), "other options"), (dict(length_required=51), "other options"),
                        (dict(adapter_fasta=fa[::-1]), "another adapter list"),
                        (dict(start_adapter=synth.ADAPTER_START[:-1]), "another adapter list")):
        other = Engine(Options(**dict(kw, **change)))
        refused([src.h.value, other.h.value], match=f"source 1 was created with {why}")
    with pytest.raises(FplError, match="other options"):
        dst.merge(Engine(Options(**dict(kw, disable_quality_filtering=True))))
    for x, y in zip(before, words(dst, dst.cycles)):
        np.testing.assert_array_equal(x, y)
    dst.merge(Engine(Options(**kw)))       # the same options built anew are accepted


def test_source_on_another_device_is_refused():
    if EMULATED:
        pytest.skip("the emulator has one device")
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    dst, other = engine(Options(start_adapter=synth.ADAPTER_START)), engine(Options(start_adapter=synth.ADAPTER_START, device=1))
    with pytest.raises(FplError, match="device"):
        dst.merge(other)


# ---- 7. launches ----
def test_one_launch_per_merge():
    opt = cases.OPTION_SETS["default_se"]
    dst, a, b = engine(opt), engine(opt), engine(opt)
    for k, e in enumerate((dst, a, b)):
        e.process(synth.ont_like(30, 1200, 70 + k))
    dst.set_timing(True)
    kt = dst.kernel_times()
    assert len(kt) == 28 and list(kt)[-1] == "k_merge_stats"
    before = dst.launch_count
    dst.merge(a, b)
    dst.sync()
    assert dst.launch_count == before + 1 and dst.kernel_times()["k_merge_stats"][1] == 1
    dst.merge(a)
    dst.sync()
    assert dst.launch_count == before + 2 and dst.kernel_times()["k_merge_stats"][1] == 2
