"""TEST INFRASTRUCTURE: fastplong's JSON report (JsonReporter::report, reference src/jsonreporter.cpp:11-94) restated in plain
Python from downloaded accumulators — the two Stats blocks (include/fplgpu.h layout, any capacity), the FilterResult counter
block and the Options — with Python's '%g' for every double (correctly rounded, half to even: the same text as glibc's
"%.6g" and libstdc++'s default ostream << double).  It shares no code with fpl_report_json; the GPU tests compare the
library's report with it on inputs that have no golden run, and tests/test_report_json.py pins it to the reference's own
reports.  Not used by the product path."""
import numpy as np

from fastplong_b200 import abi


def _g(v):
    return "%g" % v


def _ratio(a, b):
    return 0.0 if b == 0 else float(a) / float(b)       # (double)a / (double)b, as the reference divides


def summarize(block):
    """Stats::summarize (src/stats.cpp:150-256) of one block: scalars and the 11 curves (float64 arrays)."""
    block = np.asarray(block, dtype=np.int64)
    C = (block.shape[0] - abi.STATS_TAIL) // 16
    content = block[:8 * C].reshape(8, C)
    qual = block[8 * C:16 * C].reshape(8, C)
    tail = block[16 * C:]
    tot = content.sum(axis=0)
    zero = np.flatnonzero(tot == 0)
    T = int(zero[0]) if len(zero) else C              # the first cycle with no base; all of them without one
    qh = tail[abi.STATS_QUALHIST:abi.STATS_QUALHIST + 128]
    reads = int(tail[abi.STATS_READS])
    s = {"reads": reads, "bases": int(tot[:T].sum()), "q20": int(qh[33 + 20:127].sum()), "q30": int(qh[33 + 30:127].sum()),
         "gc": int(content[ord("G") & 7, :T].sum() + content[ord("C") & 7, :T].sum()), "cycles": T,
         "mean_length": int(tail[abi.STATS_LENSUM]) // reads if reads else 0, "kmer": tail[abi.STATS_KMER:abi.STATS_KMER + 1024]}
    totf = tot[:T].astype(np.float64)
    mean = qual[:, :T].sum(axis=0).astype(np.float64) / totf
    bins = [ord(x) & 7 for x in "ATUCGN"]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = {b: np.where(content[b, :T] == 0, mean, qual[b, :T].astype(np.float64) / content[b, :T].astype(np.float64))
             for b in bins}
    s["quality"] = q.__getitem__
    s["mean"] = mean
    cc = {b: content[b, :T].astype(np.float64) / totf for b in bins}
    s["content"] = cc.__getitem__
    s["gc_curve"] = (content[ord("G") & 7, :T] + content[ord("C") & 7, :T]).astype(np.float64) / totf
    return s


def _curve(a):
    return ",".join(map(_g, np.asarray(a, dtype=np.float64).tolist()))


def _stats_json(key, s, is_rna):
    t = "U" if is_rna else "T"
    out = [f'\t"{key}": {{\n',
           f'\t\t"total_reads": {s["reads"]},\n', f'\t\t"total_bases": {s["bases"]},\n', f'\t\t"q20_bases": {s["q20"]},\n',
           f'\t\t"q30_bases": {s["q30"]},\n', f'\t\t"total_cycles": {s["cycles"]},\n', '\t\t"quality_curves": {\n']
    qual = [("A", s["quality"](ord("A") & 7)), (t, s["quality"](ord(t) & 7)), ("C", s["quality"](ord("C") & 7)),
            ("G", s["quality"](ord("G") & 7)), ("mean", s["mean"])]
    out.append(",\n".join(f'\t\t\t"{n}":[{_curve(v)}]' for n, v in qual) + "\n")
    out.append("\t\t},\n\t\t\"content_curves\": {\n")
    cont = [(n, s["content"](ord(n) & 7)) for n in ("A", t, "C", "G", "N")] + [("GC", s["gc_curve"])]
    out.append(",\n".join(f'\t\t\t"{n}":[{_curve(v)}]' for n, v in cont) + "\n")
    out.append("\t\t},\n\t\t\"kmer_count\": {\n")
    letters = "A" + t + "CG"
    lines = []
    for i in range(64):
        first = letters[(i >> 4) & 3] + letters[(i >> 2) & 3] + letters[i & 3]
        lines.append(",".join(f'\t\t\t"{first}{letters[(j >> 2) & 3]}{letters[j & 3]}":{int(s["kmer"][(i << 4) + j])}'
                              for j in range(16)))
    out.append(",\n".join(lines) + "\n")
    out.append("\t\t}\n\t},\n")
    return "".join(out)


def adapter_counts(counters, adapters):
    """FilterResult::mAdapter from the event table (substrings folded over the adapters), in classcomp order"""
    width = abi.MAX_ADAPTER_LEN + 1
    table = np.asarray(counters[abi.CNT_FIXED:abi.CNT_FIXED + len(adapters) * 2 * width]).reshape(len(adapters), 2, width)
    m = {}
    for idx, side, c in zip(*np.nonzero(table)):
        a = adapters[idx]
        if c == 0 or c > len(a):
            continue
        key = a[len(a) - c:] if side == 0 else a[:c]
        m[key] = m.get(key, 0) + int(table[idx, side, c])
    return sorted(m.items(), key=lambda kv: (len(kv[0]), kv[0].encode()))


def report(pre, post, counters, options, command="", version="0.4.1", is_rna=False):
    """The report text (bytes) JsonReporter::report writes for these accumulators."""
    b = [summarize(pre), summarize(post)]
    cnt = np.asarray(counters, dtype=np.int64)
    o = []
    o.append("{\n\t\"summary\": {\n")
    o.append(f'\t\t"fastplong_version": "{version}",\n')
    for key, s, close in (("before_filtering", b[0], "\t\t},\n"), ("after_filtering", b[1], "\t\t}\n")):
        o.append(f'\t\t"{key}": {{\n')
        o.append(f'\t\t\t"total_reads":{s["reads"]},\n\t\t\t"total_bases":{s["bases"]},\n')
        o.append(f'\t\t\t"q20_bases":{s["q20"]},\n\t\t\t"q30_bases":{s["q30"]},\n')
        o.append(f'\t\t\t"q20_rate":{_g(_ratio(s["q20"], s["bases"]))},\n\t\t\t"q30_rate":{_g(_ratio(s["q30"], s["bases"]))},\n')
        o.append(f'\t\t\t"read_mean_length":{s["mean_length"]},\n\t\t\t"gc_content":{_g(_ratio(s["gc"], s["bases"]))}\n')
        o.append(close)
    o.append("\t},\n")
    f = cnt[abi.CNT_FILTER:abi.CNT_FILTER + 32]
    o.append("\t\"filtering_result\": {\n")
    o.append(f'\t\t"passed_filter_reads": {f[abi.PASS_FILTER]},\n\t\t"low_quality_reads": {f[abi.FAIL_QUALITY]},\n')
    o.append(f'\t\t"too_many_N_reads": {f[abi.FAIL_N_BASE]},\n')
    if options.low_complexity_filter:
        o.append(f'\t\t"low_complexity_reads": {f[abi.FAIL_COMPLEXITY]},\n')
    o.append(f'\t\t"too_short_reads": {f[abi.FAIL_LENGTH]},\n\t\t"too_long_reads": {f[abi.FAIL_TOO_LONG]}\n')
    o.append("\t},\n")
    ads = options.adapter_list()
    if not options.disable_adapter_trimming and (ads[0] or ads[1]):
        name = lambda a: "unspecified" if a in ("", "auto") else a  # noqa: E731
        o.append("\t\"adapter_cutting\": {\n")
        o.append(f'\t\t"adapter_trimmed_reads": {cnt[abi.CNT_ADAPTER_READS]},\n')
        o.append(f'\t\t"adapter_trimmed_bases": {cnt[abi.CNT_ADAPTER_BASES]},\n')
        o.append(f'\t\t"read_start_adapter": "{name(ads[0])}",\n\t\t"read_end_adapter": "{name(ads[1])}",\n')
        items = adapter_counts(cnt, ads)
        total = sum(v for _, v in items)
        shown = [(k, v) for k, v in items if total and not (v / float(total) < 0.01)]
        parts = [f'"{k}":{v}' for k, v in shown]
        if total - sum(v for _, v in shown) > 0:
            parts.append(f'"others":{total - sum(v for _, v in shown)}')
        o.append('\t\t"read_adapter_counts": {' + ", ".join(parts) + "}\n\t},\n")
    if options.trim_poly_x:
        o.append("\t\"polyx_trimming\": \t{\n")
        for i, key in enumerate(("polyx_trimmed_reads", "polyx_trimmed_bases")):
            v = cnt[(abi.CNT_POLYX_BASES if i else abi.CNT_POLYX_READS):][:4]
            o.append(f'\t\t"total_{key}": {int(v.sum())},\n')
            o.append(f'\t\t"{key}":{{"A": {v[0]}, "T": {v[1]}, "C": {v[2]}, "G": {v[3]}}}' + ("\n\t},\n" if i else ",\n"))
    o.append(_stats_json("read_before_filtering", b[0], is_rna))
    o.append(_stats_json("read_after_filtering", b[1], is_rna))
    o.append(f'\t"command": "{command}"\n}}')
    return "".join(o).encode()


def without_command(text):
    """the report minus its "command" line, as the golden fixtures' json_text_md5 hashes it"""
    return b"\n".join(ln for ln in text.split(b"\n") if b'"command"' not in ln)
