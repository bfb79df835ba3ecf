"""fpl_state_export / fpl_state_merge (Engine.export_state / merge_state, distributed.gather_engine): a context's state as a byte
image, merged into another context with fpl_merge_stats' semantics:
  - round trip: an image merged into a fresh context gives the same image, Stats words, counters and both reports;
  - equivalence: shards merged as live contexts (fpl_merge_stats) and as images leave equal images and reports, for a destination
    holding data, a source longer than it, a destination reserved far above, empty sources, an image twice, capture off and
    processing after the merge;
  - the reference: contiguous shards of the html_golden runs, each processed in a process of its own that writes an image file,
    merged in this one, give the -w 1 reports (golden md5s; fresh runs where oracle/_ref/fastplong_ref is built);
  - refusals leave the destination's image unchanged; the two-phase export; one k_merge_stats launch per call; images past
    k_merge_stats' grid cap;
  - gather_engine over gloo with two processes sharing one GPU, and over NCCL with one rank per GPU (two GPUs)."""
import ctypes as C
import dataclasses
import hashlib
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:            # run as a script (the shard and NCCL workers below)
    sys.path.insert(0, ROOT)

import capacity  # noqa: E402
import cases  # noqa: E402
import html_golden  # noqa: E402
import report_twin  # noqa: E402
import test_gpu_merge as M  # noqa: E402
from fastplong_b200 import Options, abi, pack_reads, synth  # noqa: E402
from fastplong_b200.binding import Engine, FplError  # noqa: E402
from oracle_lib import REF_BIN  # noqa: E402

pytestmark = pytest.mark.gpu

EMULATED = os.environ.get("FPL_EMULATE", "") not in ("", "0")
TIME = html_golden.TIME
engine = M.engine
HEADER = 248                                   # FPL_STATE_HEADER_BYTES
FIELDS = ("magic", "format", "abi", "total", "n_adapters", "adapter_bytes", "counter_words", "rows", "used_cycles",
          "reduced_rows", "keep", "complete", "merged", "n_pre", "n_post")


def header(img):
    return dict(zip(FIELDS, struct.unpack_from("<15q", img)))


def sections(img):
    """the byte offsets where the image's sections start, and its end"""
    h = header(img)
    at = [HEADER, HEADER + h["adapter_bytes"]]
    sw = 8 * abi.stats_words(h["rows"])
    for n in (sw, sw, 8 * h["counter_words"], 8 * h["n_pre"], 8 * h["n_post"]):
        at.append(at[-1] + n)
    assert at[-1] == h["total"] == len(img)
    return at


def state(e, is_rna=False, html=True):
    """everything a context's reports depend on: its image, JSON and HTML (or the HTML refusal's message)"""
    try:
        text = e.report_html(time_text=TIME, is_rna=is_rna) if html else None
    except FplError as x:
        text = str(x)
    return e.export_state(), e.report_json(is_rna=is_rna), text


def both_ways(make_dst, srcs, is_rna=False):
    """the sources merged into one destination as contexts and into another as images: their states must be equal"""
    live, img = make_dst(), make_dst()
    live.merge(*srcs)
    img.merge_state(*[s.export_state() for s in srcs])
    got, want = state(img, is_rna), state(live, is_rna)
    assert header(got[0]) == header(want[0])
    for a, b, what in zip(got, want, ("image", "JSON report", "HTML report")):
        M.assert_same(a, b, what)
    return img


# ---- 1. round trip ----
@pytest.mark.parametrize("name", sorted(M.SHARD_SETS))
def test_round_trip(name):
    opt, batch, rna = M.SHARD_SETS[name], M.shard_batch(name), name.startswith("rna")
    a = engine(opt)
    a.process(batch)
    img = a.export_state()
    h = header(img)
    assert h["rows"] == h["used_cycles"] == int(batch.lens.max()) and (h["keep"], h["complete"], h["merged"]) == (1, 1, 0)
    assert h["n_pre"] == batch.n_reads and len(img) % 8 == 0
    b = engine(opt)
    b.merge_state(img)
    assert b.export_state() == img
    M.assert_equal_contexts(b, a, rna)
    c = engine(opt)                         # bytearray and numpy images are the same image
    c.merge_state(bytearray(img), np.frombuffer(img, np.uint8))
    d = engine(opt)
    d.merge(a, a)
    assert c.export_state() == d.export_state()


# ---- 2. equivalence with fpl_merge_stats ----
@pytest.mark.parametrize("name", sorted(M.SHARD_SETS))
def test_shards_into_a_destination_holding_data(name):
    opt, batch, rna = M.SHARD_SETS[name], M.shard_batch(name), name.startswith("rna")
    reads = M.reads_of(batch)
    cut = np.linspace(0, len(reads), 4).astype(int)
    parts = [pack_reads(reads[a:b]) for a, b in zip(cut[:-1], cut[1:])]
    srcs = [engine(opt) for _ in parts[1:]]
    for s, p in zip(srcs, parts[1:]):
        s.process(p)

    def dst():
        e = engine(opt)
        e.process(parts[0])
        return e
    got = both_ways(dst, srcs, rna)
    whole = engine(opt)
    whole.process(batch)
    M.assert_equal_contexts(got, whole, rna)
    assert got.export_state() == whole.export_state()


def test_source_longer_than_the_destination():
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    short, long = pack_reads(M.long_reads(1, [120, 300, 250] * 5)), pack_reads(M.long_reads(2, [350, 2000, 7777, 5000] * 3))
    src = engine(opt)
    src.process(long)

    def dst():
        e = engine(opt)
        e.process(short)
        return e
    got = both_ways(dst, [src])
    assert got.cycles >= 7777 and header(got.export_state())["rows"] == 7777


def test_destination_reserved_far_above():
    opt = cases.OPTION_SETS["default_se"]
    src = engine(opt)
    src.process(synth.ont_like(40, 900, 12))

    def dst():
        e = engine(opt)
        e.reserve_cycles(1 << 16)
        e.process(synth.ont_like(40, 1500, 11))
        return e
    got = both_ways(dst, [src])
    assert got.cycles == 1 << 16


def test_empty_sources_and_the_same_image_twice():
    opt = cases.OPTION_SETS["fasta64_polyx"]
    src, empty = engine(opt), engine(opt)
    src.process(cases.hifi_fasta64_batch(22, n=40, mean=1200))
    h = header(empty.export_state())
    assert h["rows"] == h["n_pre"] == h["n_post"] == 0
    both_ways(lambda: engine(opt), [empty])                 # rows == 0 only
    both_ways(lambda: engine(opt), [empty, src, empty])
    both_ways(lambda: engine(opt), [src, src])

    def dst():
        e = engine(opt)
        e.process(cases.hifi_fasta64_batch(23, n=20, mean=900))
        return e
    before = dst().export_state()
    d = dst()
    d.merge_state()                                         # no image: nothing changes
    d.merge_state(empty.export_state())                     # an empty image adds nothing
    assert d.export_state() == before


def test_capture_off():
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    a, b = synth.ont_like(40, 1500, 51), synth.ont_like(40, 1500, 52)
    src = engine(opt, keep=False)
    src.process(b)
    assert header(src.export_state())["complete"] == 0

    def dst():
        e = engine(opt)
        e.process(a)
        return e
    got = both_ways(dst, [src])
    with pytest.raises(FplError, match="capture"):
        got.report_html(time_text=TIME)
    got = both_ways(lambda: engine(opt, keep=False), [engine(opt)])      # a destination with capture off takes no list
    assert header(got.export_state())["complete"] == 0


def test_merged_flag_travels():
    """an image whose context was all-reduced over several ranks (its `merged` word set: a real one needs two GPUs, test 9) makes
    the destination refuse the HTML report and keep the JSON one, and the flag goes on into the destination's own image"""
    opt = cases.OPTION_SETS["default_se"]
    src = engine(opt)
    src.process(synth.ont_like(30, 1200, 55))
    img = bytearray(src.export_state())
    struct.pack_into("<q", img, 8 * FIELDS.index("merged"), 1)
    dst = engine(opt)
    dst.merge_state(bytes(img))
    with pytest.raises(FplError, match="several ranks"):
        dst.report_html(time_text=TIME)
    assert dst.report_json() == src.report_json() and header(dst.export_state())["merged"] == 1


def test_processing_after_the_merge_continues_the_sequence():
    opt = cases.MASK_BREAK_SETS["mask_and_break"]
    b1, b2, b3 = (cases.blocky_quality_batch(30 + k, n=40) for k in range(3))
    src = engine(opt)
    src.process(b2)
    live, img = engine(opt), engine(opt)
    for e in (live, img):
        e.process(b1)
    live.merge(src)
    img.merge_state(src.export_state())
    whole = engine(opt)
    for e in (live, img):
        e.process(b3)
    for b in (b1, b2, b3):
        whole.process(b)
    assert img.export_state() == live.export_state() == whole.export_state()
    M.assert_equal_contexts(img, whole)


# ---- 3. the reference: shards processed in processes of their own ----
def shard_worker(name, k, n_shards, path):
    """shard k of the html_golden run `name`, processed in this process, its image written to `path`"""
    if EMULATED:
        import simt_emu
        from fastplong_b200 import binding
        binding.LIB_PATH = simt_emu.build_library()
    from fastplong_b200 import distributed as D
    opt, batch = html_golden.run_input(name)
    mine, _ = D.shard(batch, k, n_shards)
    e = engine(opt)
    e.process(mine)
    with open(path, "wb") as f:
        f.write(e.export_state())


def golden_json_md5(name):
    """the -j report's md5 (minus the command) the reference wrote for this run: the same at every -w (merge_golden.json)"""
    g = json.load(open(M.FIXTURE)).get(name)
    return None if g is None else set(g["json_md5"].values())


@pytest.mark.parametrize("name", sorted(html_golden.RUNS))
def test_shard_images_match_the_reference(name, tmp_path):
    opt, batch = html_golden.run_input(name)
    rna = name in html_golden.IS_RNA
    n_shards = 3
    paths = [str(tmp_path / f"shard{k}.img") for k in range(n_shards)]
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "shard", name, str(k), str(n_shards), paths[k]], cwd=ROOT,
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for k in range(n_shards)]
    for p in procs:
        out, err = p.communicate(timeout=900)
        assert p.returncode == 0, err[-3000:]
    images = [open(q, "rb").read() for q in paths]
    assert all(header(im)["n_pre"] for im in images)
    dst = engine(opt)
    dst.merge_state(*images)
    html = dst.report_html(command="fastplong -i in.fq", title=html_golden.TITLE.get(name, "fastplong report"), time_text=TIME,
                           is_rna=rna)
    js = report_twin.without_command(dst.report_json(is_rna=rna))
    whole = engine(opt)
    whole.process(batch)
    assert dst.export_state() == whole.export_state()
    empty = html_golden.empties(*M.twin_lists(opt, [batch]))
    g = json.load(open(html_golden.FIXTURE))[name]
    checked = False
    if g["input_md5"] == html_golden.input_md5(batch):
        assert html_golden.masked_md5(html, empty) == g["html_md5"]
        if golden_json_md5(name):
            assert hashlib.md5(js).hexdigest() in golden_json_md5(name)
        checked = True
    if os.path.exists(REF_BIN):
        ref_html = html_golden.run_reference(REF_BIN, name, str(tmp_path))
        M.assert_same(html_golden.mask(html, empty), html_golden.mask(ref_html, empty), "masked HTML report")
        M.assert_same(js, report_twin.without_command(open(tmp_path / "r.json", "rb").read()), "JSON report")
        checked = True
    if not checked:
        pytest.skip("no reference binary, and numpy made another input than when the fixture was made")


# ---- 4. refusals ----
def test_refusals_leave_the_destination_unchanged():
    opt = cases.OPTION_SETS["fasta5"]
    b = pack_reads(cases.planted_fasta_reads(61, n=40))
    dst, src = engine(opt), engine(opt)
    dst.process(b)
    src.process(synth.ont_like(30, 1200, 62))
    img = src.export_state()
    before = dst.export_state()
    lib = dst.lib

    def refused(image, match=""):
        with pytest.raises(FplError, match=match):
            dst.merge_state(img, image)
        assert dst.export_state() == before

    def with_word(k, v):
        x = bytearray(img)
        struct.pack_into("<q", x, 8 * k, v)
        return bytes(x)
    for k, f in enumerate(FIELDS):                          # every header word corrupted in turn
        refused(with_word(k, -1), "image 1")
    refused(with_word(1, 2), "image format 2")
    refused(with_word(2, abi.ABI_VERSION + 1), "FPL_ABI_VERSION")
    refused(with_word(7, header(img)["rows"] + 1), "rows")
    refused(with_word(10, 2), "flag")
    for at in sections(img):                                # truncated at every section boundary and one byte short of it
        for n in (at, at - 1):
            if n < len(img):
                refused(img[:n], "truncated" if n < HEADER else "bytes")
    refused(img + b"\0", "trailing")
    # the options: each field of the block changed, and engines made with other options in every class
    fields = [n for n, _ in abi.FplOptions._fields_][2:-1]
    assert img[120:244] == bytes(src._keep[0])[8:132] and img[244:248] == b"\0" * 4       # no device in the image
    for name in fields:
        x = bytearray(img)
        off = 120 + getattr(abi.FplOptions, name).offset - 8
        x[off] ^= 1
        refused(bytes(x), "other options")
    fa = opt.adapter_fasta
    kw = dict(start_adapter=synth.ADAPTER_START, adapter_fasta=fa, trim_poly_x=True, poly_x_min_len=8)
    for change in (dict(trim_front=3), dict(cut_front=True), dict(poly_x_min_len=9), dict(disable_adapter_trimming=True),
                   dict(disable_quality_filtering=True), dict(length_required=51), dict(low_complexity_filter=True),
                   dict(mask=True), dict(break_reads=True)):
        refused(Engine(Options(**dict(kw, **change))).export_state(), "other options")
    for change in (dict(adapter_fasta=fa[::-1]), dict(start_adapter=synth.ADAPTER_START[:-1]), dict(adapter_fasta=fa[:-1])):
        refused(Engine(Options(**dict(kw, **change))).export_state(), "another adapter list")
    x = bytearray(img)                                      # an adapter's bytes, and its length word
    x[HEADER + 8] ^= 2
    refused(bytes(x), "another adapter list")
    refused(with_word(HEADER // 8, 3), "another adapter list")
    # null and negative arguments
    ptr = np.frombuffer(img, np.uint8)

    def raw(d, images, sizes, n, match):
        assert lib.fpl_state_merge(d, images, sizes, n) < 0
        assert match in lib.fpl_last_error().decode(), lib.fpl_last_error().decode()
        assert dst.export_state() == before
    one = (C.c_void_p * 1)(ptr.ctypes.data)
    size = (C.c_int64 * 1)(len(img))
    raw(None, one, size, 1, "null destination")
    raw(dst.h, None, size, 1, "null image")
    raw(dst.h, one, None, 1, "null image")
    raw(dst.h, one, size, -1, "negative number")
    raw(dst.h, (C.c_void_p * 1)(None), size, 1, "image 0 is null")
    raw(dst.h, one, (C.c_int64 * 1)(-5), 1, "negative size")
    n = C.c_int64()
    assert lib.fpl_state_export(None, None, 0, C.byref(n)) < 0 and lib.fpl_state_export(dst.h, None, 0, None) < 0
    dst.merge_state(Engine(Options(**kw)).export_state())  # the same options built anew are accepted
    assert dst.export_state() == before


# ---- 5. two-phase export ----
def test_two_phase_export():
    e = engine(cases.OPTION_SETS["default_se"])
    e.process(synth.ont_like(20, 1000, 81))
    img = e.export_state()
    lib, n = e.lib, C.c_int64()
    assert lib.fpl_state_export(e.h, None, 0, C.byref(n)) == 1 and n.value == len(img)
    for cap in (0, len(img) - 1):
        canary = np.full(len(img) + 64, 0xA5, np.uint8)
        n.value = -1
        assert lib.fpl_state_export(e.h, canary.ctypes.data, cap, C.byref(n)) == 1
        assert n.value == len(img) and (canary == 0xA5).all()
    out = np.full(len(img) + 64, 0xA5, np.uint8)
    assert lib.fpl_state_export(e.h, out.ctypes.data, len(img), C.byref(n)) == 0
    assert out[:len(img)].tobytes() == img and (out[len(img):] == 0xA5).all()


# ---- 6. launches ----
def test_one_launch_per_merge():
    opt = cases.OPTION_SETS["default_se"]
    srcs = [engine(opt) for _ in range(3)]
    for k, e in enumerate(srcs):
        e.process(synth.ont_like(10, 600 + 300 * k, 90 + k))
    images = [e.export_state() for e in srcs]
    dst = engine(opt)
    dst.set_timing(True)
    for k, n in enumerate((1, 3, 8)):
        before = dst.launch_count
        dst.merge_state(*[images[i % 3] for i in range(n)])
        assert dst.launch_count == before + 1 and dst.kernel_times()["k_merge_stats"][1] == k + 1
    want = engine(opt)
    want.merge(*[srcs[i % 3] for i in (0, 0, 1, 2, 0, 1, 2, 0, 1, 2, 0, 1)])
    assert dst.export_state() == want.export_state()


# ---- 7. capacities ----
def test_images_past_the_merge_cap():
    """images of 1024 (rows == C), 2048 and 16384 cycles (more words than k_merge_stats' capped grid has threads), into an empty
    and into a 2048-cycle destination; the list boundaries fall inside HTML_CHUNK chunks"""
    K = capacity.constants()
    batches = capacity.merge_sources(K, seed=9)
    if EMULATED and sum(int(b.lens.sum()) for b in batches) // 100 > 20000:
        pytest.skip("too slow for the emulator")
    opt = capacity.REPORT_OPT
    srcs = [engine(opt) for _ in batches]
    for e, b in zip(srcs, batches):
        e.process(b)
    assert sorted(e.cycles for e in srcs) == [1024, 2048, 16384]
    assert 2 * 16 * int(max(batches[2].lens)) > K["k_merge_stats_BLOCKS"] * 256
    got = both_ways(lambda: engine(opt), srcs)
    whole = engine(opt)
    _, lists = capacity.report_run(whole, opt, batches, "state/whole")
    capacity.check_reports(got, opt, lists, "state/fresh")

    def dst():
        e = engine(opt)
        e.process(batches[1])
        return e
    got = both_ways(dst, [srcs[0], srcs[2]])
    whole = engine(opt)
    _, lists = capacity.report_run(whole, opt, [batches[1], batches[0], batches[2]], "state/whole2")
    capacity.check_reports(got, opt, lists, "state/into")


# ---- 8. processes sharing one GPU: gather_engine over gloo ----
GLOO_OPT, GLOO_N = "mask_and_break", 90


def gloo_batch():
    return cases.blocky_quality_batch(95, n=GLOO_N)


def gloo_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    if EMULATED:
        import simt_emu
        from fastplong_b200 import binding
        binding.LIB_PATH = simt_emu.build_library()
    import torch.distributed as dist
    from fastplong_b200 import distributed as D
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    opt = cases.MASK_BREAK_SETS[GLOO_OPT]
    mine, _ = D.shard(gloo_batch(), rank, world)
    for root in range(world):                # each rank in turn the root: rank order either way
        e = engine(opt)
        e.process(mine)
        own = e.export_state()
        D.gather_engine(e, root=root)
        if rank == root:
            open(os.path.join(out_dir, f"root{root}.img"), "wb").write(e.export_state())
            open(os.path.join(out_dir, f"root{root}.html"), "wb").write(e.report_html(time_text=TIME))
        else:
            assert e.export_state() == own
    # a rank with other options: root 1 refuses rank 0's image and is left with its own state
    e = engine(opt if rank == 1 else cases.MASK_BREAK_SETS["mask_default"])
    e.process(mine)
    own = e.export_state()
    try:
        D.gather_engine(e, root=1)
        refused = False
    except FplError:
        refused = True
    if rank == 1:
        assert refused and e.export_state() == own
        open(os.path.join(out_dir, "refused"), "w").write("ok")
    dist.barrier()
    dist.destroy_process_group()


def test_gather_engine_two_processes_one_gpu(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.spawn(gloo_worker, args=(2, 31000 + os.getpid() % 2000, str(tmp_path)), nprocs=2, join=False)
    deadline = time.monotonic() + 900
    try:
        while not ctx.join(timeout=5):
            assert time.monotonic() < deadline, "the ranks did not finish in time"
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.kill()
            p.join(30)
    assert not any(p.is_alive() for p in ctx.processes)
    opt = cases.MASK_BREAK_SETS[GLOO_OPT]
    whole = engine(opt)
    whole.process(gloo_batch())
    for root in range(2):
        assert open(tmp_path / f"root{root}.img", "rb").read() == whole.export_state()
        M.assert_same(open(tmp_path / f"root{root}.html", "rb").read(), whole.report_html(time_text=TIME), "HTML report")
    assert (tmp_path / "refused").exists()


# ---- 9. two GPUs ----
def n_gpus():
    if EMULATED:
        return 1
    import torch
    return torch.cuda.device_count()


def test_image_from_another_device():
    if n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    opt = cases.OPTION_SETS["cut_polyx_cplx"]
    b = synth.ont_like(60, 1500, 97)
    src = engine(opt)
    src.process(b)
    dst = engine(dataclasses.replace(opt, device=1))
    with pytest.raises(FplError, match="device"):
        dst.merge(src)
    dst.merge_state(src.export_state())
    assert dst.export_state() == src.export_state()
    M.assert_equal_contexts(dst, src)


def nccl_worker():
    """one rank per GPU under torch.distributed.run: gather_engine over NCCL (CUDA uint8 tensors) to rank 0 gives one engine's
    reports over the whole batch; after a multi-rank fpl_allreduce_stats the merged flag travels in the images, and rank 0's
    destination then refuses the HTML report exactly as after fpl_merge_stats of that context"""
    import torch
    import torch.distributed as dist
    from fastplong_b200 import distributed as D
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    opt = dataclasses.replace(cases.OPTION_SETS["cut_polyx_cplx"], device=local)
    batch = synth.ont_like(200, 2000, 98, p_chimera=0.05)
    mine, _ = D.shard(batch, rank, world)
    e = engine(opt)
    e.process(mine)
    D.gather_engine(e)
    red = engine(opt)
    red.process(mine)
    D.init_engine_comm(red, rank, world)
    D.merge_engine(red)
    red.sync()
    img = red.export_state()
    assert header(img)["merged"] == 1
    live, imaged = engine(opt), engine(opt)
    live.merge(red)
    imaged.merge_state(img)
    assert imaged.export_state() == live.export_state()
    D.gather_engine(red)
    if rank == 0:
        whole = engine(opt)
        whole.process(batch)
        assert e.export_state() == whole.export_state()
        M.assert_equal_contexts(e, whole)
        for d in (live, imaged, red):
            with pytest.raises(FplError, match="several ranks"):
                d.report_html(time_text=TIME)
        print("NCCL_GATHER_OK")
    dist.barrier()
    dist.destroy_process_group()


def test_gather_engine_one_rank_per_gpu():
    if n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(29900 + os.getpid() % 300), os.path.abspath(__file__), "nccl"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    assert "NCCL_GATHER_OK" in p.stdout


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    if sys.argv[1] == "shard":
        shard_worker(sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), sys.argv[5])
    else:
        nccl_worker()
