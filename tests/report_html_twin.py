"""TEST INFRASTRUCTURE: fastplong's HTML report (HtmlReporter::report, reference src/htmlreporter.cpp:75-253, with the
Stats::reportHtml* functions of src/stats.cpp:550-1011) restated in plain Python from downloaded accumulators — the two Stats
blocks, the FilterResult counters, the Options — and the two per-read lists Stats::statRead builds (the oracle's records and
output reads give them).  It shares no code with fpl_report_html.  Doubles divide as numpy float64 (IEEE, like the reference)
and print like glibc: '%f' / '%g', with the sign of a NaN shown ("-nan").  The entries the reference leaves uninitialised
(quirk 1 of the density arrays) are 0, as the library defines them.  Not used by the product path."""
import math

import numpy as np

import report_twin
from fastplong_b200 import abi


def _nan_sign(v, text):
    if math.isnan(v):
        return "-nan" if math.copysign(1.0, v) < 0 else "nan"
    return text


def f_str(v):
    """std::to_string(double)"""
    v = float(v)
    return _nan_sign(v, "%f" % v)


def g_str(v):
    """ostream << double"""
    v = float(v)
    return _nan_sign(v, "%g" % v)


def div(a, b):
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(a) / np.float64(b))


def format_number(number):
    num = float(number)
    order = 0
    while num > 1000.0:
        order += 1
        num /= 1000.0
    return str(int(number)) if order == 0 else f_str(num) + " " + ["", "K", "M", "G", "T", "P"][order]


def get_percents(a, b):
    return "0.0" if b == 0 else f_str(div(float(a) * 100.0, b))


def row(k, v):
    return f"<tr><td class='col1'>{k}</td><td class='col2'>{v}</td></tr>\n"


def read_lists(lens, records, segments=None):
    """the lists one fpl_process_* call appends: every input read (length, pre_median_qual); every passing output read in
    input order, then segment order (the records' segments, or the --mask/--break output-read list)"""
    pre = [(int(lens[i]), int(records[i]["pre_median_qual"])) for i in range(len(records))]
    post = []
    if segments is not None:
        post = [(int(s["len"]), int(s["median_qual"])) for s in segments if s["result"] == abi.PASS_FILTER]
    else:
        for r in records:
            for k in range(int(r["n_segments"])):
                if r["seg_result"][k] == abi.PASS_FILTER:
                    post.append((int(r["seg_len"][k]), int(r["seg_median_qual"][k])))
    return pre, post


def length_stats(lst, lensum):
    """Stats::calcLengthHistogram: min, max, median, N50 (int * int products wrapped to 32 bits)"""
    hist = {}
    for L, _ in lst:
        hist[L] = hist.get(L, 0) + 1
    if not hist:
        return 0, 0, 0, 0
    total, readnum, n50, med = 0, 0, 0, 0
    for L in sorted(hist):
        p = (L * hist[L]) & 0xFFFFFFFF
        total += p - (1 << 32) if p >= 1 << 31 else p
        if n50 == 0 and total > lensum // 2:
            n50 = L
        readnum += hist[L]
        if med == 0 and readnum > len(lst) // 2:
            med = L
        if med > 0 and n50 > 0:
            break
    return min(hist), max(hist), med, n50


def curve_x(cycles):
    if cycles <= 300:
        return list(range(1, cycles + 1))
    x = list(range(1, 41))
    pos = 40.0
    while True:
        pos *= 1.05
        if pos >= cycles:
            break
        x.append(int(pos))
    if x[-1] != cycles:
        x.append(cycles)
    return x


def sampled(curve, x):
    out = []
    for i, end in enumerate(x):
        start = x[i - 1] if i else 0
        total = 0.0
        for k in range(start, end):
            total += float(curve[k])
        out.append("0.0" if end == start else g_str(total / (end - start)))
    return ",".join(out)


def _basic(t, s, lst):
    tail = s["tail"]
    qh = tail[abi.STATS_QUALHIST:abi.STATS_QUALHIST + 128]
    q = {}
    acc = int(qh[40 + 33:127].sum())
    q[40] = acc
    for lo, hi in ((30, 40), (20, 30), (15, 20), (10, 15), (7, 10), (5, 7)):
        acc += int(qh[lo + 33:hi + 33].sum())
        q[lo] = acc
    mn, mx, med, n50 = length_stats(lst, int(tail[abi.STATS_LENSUM]))
    reads, bases = s["reads"], s["bases"]
    o = [f"<div class='subsection_title'>{t}: Basic statistics</div>\n", "<table>\n",
         row("total reads:", format_number(reads)), row("total bases:", format_number(bases)),
         row("minimum length:", format_number(mn)), row("maximum length:", format_number(mx)),
         row("median length:", format_number(med)), row("mean length:", format_number(s["mean_length"])),
         row("N50 length:", format_number(n50)), row("GC content:", get_percents(s["gc"], bases) + "%")]
    for k in (5, 7, 10, 15, 20, 30, 40):
        o.append(row(f"Q{k} bases:", format_number(q[k]) + " (" + get_percents(q[k], bases) + "%)"))
    o.append("</table>\n")
    return "".join(o)


def _median_hist(t, s):
    sub = f"{t}: Read median quality statistics"
    dv = sub.replace(" ", "_")
    tail = s["tail"]
    hist = tail[abi.STATS_MEDHIST:abi.STATS_MEDHIST + 128]
    mb = tail[abi.STATS_MEDBASES:abi.STATS_MEDBASES + 128]
    min_val = 0
    for i in range(94):
        if mb[i + 33] == 0:
            min_val += 1
        else:
            break
    max_val = 0
    for i in range(94, -1, -1):
        if mb[i + 33] > 0:
            max_val = i
            break
    offset = max(0, min_val - 1)
    total = max(0, min(94, max_val - min_val + 2))
    x = ",".join(str(i + offset) for i in range(total))
    pr = ",".join(g_str(div(float(hist[i + offset + 33]) * 100.0, s["reads"])) for i in range(total))
    pb = ",".join(g_str(div(float(mb[i + offset + 33]) * 100.0, s["bases"])) for i in range(total))
    return (f"<div class='subsection_title'>{sub}</div>\n<div id='mean_qual_length_histogram_figure'>\n"
            f"<div class='figure' id='plot_median_qual_hist_{dv}' style='height:400px;'></div>\n</div>\n"
            "\n<script type=\"text/javascript\">\n"
            f"var readNum={{x:[{x}],y:[{pr}],name: '% reads',type:'bar',line:{{color:'rgba(128,0,128,1.0)', width:1}}\n}};\n"
            f"var baseNum={{x:[{x}],y:[{pb}],name: '% accumulated bases',type:'bar',line:{{color:'rgba(128,128,0,1.0)', width:1}}\n}};\n"
            "var data = [readNum, baseNum];;\n"
            "var layout={legend: {x: 0, y: 1.0},title:'Read median quality distribution', xaxis:{title:'read median quality score'}, "
            "yaxis:{title:'Percent (%)'}};\n"
            f"Plotly.newPlot('plot_median_qual_hist_{dv}', data, layout);\n</script>\n")


def _density(t, lst):
    sub = f"{t}: Density plot of read median quality and read length"
    dv = sub.replace(" ", "_")
    groups = {}
    for L, m in lst:
        if L > 0:
            groups.setdefault(m, []).append(L)
    xs, ys = [], []
    for m in sorted(groups):
        for L in groups[m]:
            xs.append(m - 33)
            ys.append(L)
    pad = len(lst) - len(xs)
    x = ",".join(map(str, xs + [0] * pad))
    y = ",".join(map(str, ys + [0] * pad))
    return (f"<div class='subsection_title'>{sub}</div>\n<div id='mean_qual_length_density_figure'>\n"
            f"<div class='figure' id='plot_median_qual_length_density_{dv}' style='height:400px;'></div>\n</div>\n"
            "\n<script type=\"text/javascript\">\n"
            f"var density={{x:[{x}],y:[{y}],name: '% reads',type:'histogram2dcontour',line:{{color:'rgba(128,0,128,1.0)', width:1}}\n}};\n"
            "var data = [density];\n"
            "var layout={legend: {x: 0, y: 1.0},title:' Density plot of read median quality and read length', xaxis:{title:'read median "
            "quality score'}, yaxis:{title:'Read length', type:'log'}};\n"
            f"Plotly.newPlot('plot_median_qual_length_density_{dv}', data, layout);\n</script>\n")


QCOLORS = ["rgba(128,128,0,1.0)", "rgba(128,0,128,1.0)", "rgba(0,255,0,1.0)", "rgba(0,0,255,1.0)", "rgba(20,20,20,1.0)"]
CCOLORS = ["rgba(128,128,0,1.0)", "rgba(128,0,128,1.0)", "rgba(0,255,0,1.0)", "rgba(0,0,255,1.0)", "rgba(255, 0, 0, 1.0)",
           "rgba(20,20,20,1.0)"]


def _curves(t, s, content, is_rna, base_contents):
    sub = f"{t}: " + ("base contents" if content else "quality")
    dv = sub.replace(" ", "_").replace(":", "_")
    T = s["cycles"]
    x = curve_x(T)
    xs = ",".join(map(str, x))
    tt = "U" if is_rna else "T"
    o = [f"<div class='subsection_title'>{sub}</div>\n<div id='{dv}'>\n"
         "<div class='sub_section_tips'>Value of each position will be shown on mouse over.</div>\n"
         f"<div class='figure' id='plot_{dv}'></div>\n</div>\n\n<script type=\"text/javascript\">\nvar data=["]
    if content:
        series = [(n, s["content"](ord(n) & 7)) for n in ("A", tt, "C", "G", "N")] + [("GC", s["gc_curve"])]
    else:
        series = [(n, s["quality"](ord(n) & 7)) for n in ("A", tt, "C", "G")] + [("mean", s["mean"])]
    for k, (n, curve) in enumerate(series):
        name = n
        if content:
            cnt = base_contents[ord(n) & 7] if len(n) == 1 else base_contents[ord("G") & 7] + base_contents[ord("C") & 7]
            name = f"{n}({f_str(div(float(cnt) * 100.0, s['bases']))[:5]}%)"
        o.append(f"{{x:[{xs}],y:[{sampled(curve, x)}],name: '{name}',mode:'lines',line:{{color:'{(CCOLORS if content else QCOLORS)[k]}', width:1}}\n}},")
    o.append("];\nvar layout={title:'', xaxis:{title:'position'" + (",type:'log'" if T > 300 else ""))
    o.append("}, yaxis:{title:'" + ("base content ratios" if content else "quality") + "'}};\n")
    o.append(f"Plotly.newPlot('plot_{dv}', data, layout);\n</script>\n")
    return "".join(o)


def _kmer(t, s, is_rna):
    sub = f"{t}: KMER counting"
    dv = sub.replace(" ", "_").replace(":", "_")
    letters = "A" + ("U" if is_rna else "T") + "CG"
    k2 = lambda j: letters[(j >> 2) & 3] + letters[j & 3]  # noqa: E731
    k3 = lambda i: letters[(i >> 4) & 3] + letters[(i >> 2) & 3] + letters[i & 3]  # noqa: E731
    o = [f"<div class='subsection_title'>{sub}</div>\n<div  id='{dv}'>\n"
         "<div class='sub_section_tips'>Darker background means larger counts. The count will be shown on mouse over.</div>\n"
         "<table class='kmer_table' style='width:680px;'>\n<tr><td></td>"]
    o += [f"<td style='color:#333333'>{k2(h)}</td>" for h in range(16)]
    o.append("</tr>\n")
    mean_bases = float(s["bases"] + 1) / 2048       # Stats::mKmerBufLen = 2 << (5 * 2)
    for i in range(64):
        o.append(f"<tr><td style='color:#333333'>{k3(i)}</td>")
        for j in range(16):
            val = int(s["kmer"][(i << 4) + j])
            prop = val / mean_bases
            if prop <= 0.3:
                frac = prop * 2.0
                b = int(255 - 256 * frac)
                g = int(255 * frac)
                r = int(b * frac)
            elif prop > 3.0:
                frac = 2.0 / prop
                r = int(255 - 128 * frac)
                g = int(128 * frac)
                b = int(r * frac)
            else:
                r = g = b = 196
            km = k3(i) + k2(j)
            o.append(f"<td style='background:#{r:02x}{g:02x}{b:02x}' title='{km}: {val}\n{g_str(prop)} times as mean value'>{km}</td>")
        o.append("</tr>\n")
    o.append("</table>\n</div>\n")
    return "".join(o)


CSS = ["<style type=\"text/css\">", "td {border:1px solid #dddddd;padding:5px;font-size:12px;}",
       "table {border:1px solid #999999;padding:2x;border-collapse:collapse;width:100%}", ".col1 {width:240px; font-weight:bold;}",
       ".adapter_col {width:500px; font-size:10px;}", "img {padding:30px;}",
       "#menu {font-family:Consolas, 'Liberation Mono', Menlo, Courier, monospace;}",
       "#menu a {color:#0366d6; font-size:18px;font-weight:600;line-height:28px;text-decoration:none;font-family:-apple-system, "
       "BlinkMacSystemFont, 'Segoe UI', Helvetica, Arial, sans-serif, 'Apple Color Emoji', 'Segoe UI Emoji', 'Segoe UI Symbol'}",
       "a:visited {color: #999999}", ".alignleft {text-align:left;}", ".alignright {text-align:right;}",
       ".figure {width:680px;height:600px;}", ".header {color:#ffffff;padding:1px;height:20px;background:#000000;}",
       ".section_title {color:#ffffff;font-size:20px;padding:5px;text-align:left;background:#663355; margin-top:10px;}",
       ".section_table {width:100%;}", ".subsection_title {font-size:16px;padding:5px;margin-top:10px;text-align:left;color:#663355}",
       "#container {text-align:center;padding:3px 3px 3px 10px;font-family:Arail,'Liberation Mono', Menlo, Courier, monospace;}",
       ".menu_item {text-align:left;padding-top:5px;font-size:18px;}",
       ".highlight {text-align:left;padding-top:30px;padding-bottom:30px;font-size:20px;line-height:35px;}",
       "#helper {text-align:left;border:1px dotted #fafafa;color:#777777;font-size:12px;}",
       "#footer {text-align:left;padding:15px;color:#ffffff;font-size:10px;background:#663355;font-family:Arail,'Liberation Mono', Menlo, "
       "Courier, monospace;}",
       ".kmer_table {text-align:center;font-size:8px;padding:2px;}", ".kmer_table td{text-align:center;font-size:8px;padding:0px;color:#ffffff}",
       ".sub_section_tips {color:#999999;font-size:10px;padding-left:5px;padding-bottom:3px;}", "</style>"]


def _section(sid, title, a, b):
    return (f"<div class='section_div'>\n<div class='section_title' onclick=showOrHide('{sid}')><a name='summary'>{title}</a></div>\n"
            f"<table id='{sid}' class='section_table'>\n<tr><td>\n{a}</td><td>\n{b}</td></tr>\n</table>\n</div>\n")


def report(pre, post, counters, options, pre_list, post_list, command="", version="0.4.1", title="fastplong report",
           time_text="2026-01-01      00:00:00", is_rna=False):
    """The report text (bytes) HtmlReporter::report writes at -w 1 for these accumulators and lists."""
    blocks = []
    for blk in (pre, post):
        s = report_twin.summarize(blk)
        blk = np.asarray(blk, dtype=np.int64)
        C = (blk.shape[0] - abi.STATS_TAIL) // 16
        s["tail"] = blk[16 * C:]
        s["base_contents"] = [int(v) for v in blk[:8 * C].reshape(8, C)[:, :s["cycles"]].sum(axis=1)]
        blocks.append(s)
    lists = [pre_list, post_list]
    types = ["Before filtering", "After filtering"]
    f = np.asarray(counters, dtype=np.int64)[abi.CNT_FILTER:abi.CNT_FILTER + 32]
    o = ["<html><head><meta http-equiv=\"content-type\" content=\"text/html;charset=utf-8\" />",
         f"<title>fastplong report at {time_text} </title>",
         "<script src='https://opengene.org/plotly-1.2.0.min.js'></script>\n",
         "\n<script type='text/javascript'>\n",
         "    window.Plotly || document.write('<script src=\"https://cdn.plot.ly/plotly-1.2.0.min.js\"><\\/script>')\n",
         "</script>\n", "\n<script type=\"text/javascript\">\n", "    function showOrHide(divname) {\n",
         "        div = document.getElementById(divname);\n", "        if(div.style.display == 'none')\n",
         "            div.style.display = 'block';\n", "        else\n", "            div.style.display = 'none';\n", "    }\n",
         "</script>\n"]
    o += [ln + "\n" for ln in CSS]
    o.append("</head><body><div id='container'>\n")
    o.append("<h3 style='text-align:left;'><a href='https://github.com/OpenGene/fastplong' target='_blank' style='color:#663355;"
             f"text-decoration:none;'>{title}</a><a href='https://github.com/OpenGene/fastplong' target='_blank' "
             f"style='font-size:-2;text-decoration:none;'>(fastplong version v{version})</a></h3>\n")
    o.append("<div class='section_div'>\n<div class='section_title' onclick=showOrHide('summary')><a name='summary'>Summary</a> </div>\n"
             "<div id='summary'>\n<div class='subsection_title'>Filtering result</div>\n<div id='filtering_result'>\n"
             "<table class='summary_table'>\n")
    total = float(blocks[0]["reads"])
    fr = lambda k, code: row(k, format_number(f[code]) + " (" + f_str(div(float(f[code]) * 100.0, total)) + "%)")  # noqa: E731
    o += [fr("reads passed filters:", abi.PASS_FILTER), fr("reads with low quality:", abi.FAIL_QUALITY),
          fr("reads with too many N:", abi.FAIL_N_BASE)]
    abi_opt = options.to_abi()[0]
    if abi_opt.length_filter_enabled:
        o.append(fr("reads too short:", abi.FAIL_LENGTH))
        if abi_opt.length_max > 0:
            o.append(fr("reads too long:", abi.FAIL_TOO_LONG))
    if abi_opt.complexity_enabled:
        o.append(fr("reads with low complexity:", abi.FAIL_COMPLEXITY))
    o.append("</table>\n</div>\n</div>\n</div>\n")
    o.append(_section("basic_stat", "Basic statistics", *[_basic(types[w], blocks[w], lists[w]) for w in (0, 1)]))
    o.append(_section("median_qual_stat", "Median qual histogram", *[_median_hist(types[w], blocks[w]) for w in (0, 1)]))
    o.append(_section("median_qual_length_density", "Median qual length density", *[_density(types[w], lists[w]) for w in (0, 1)]))
    o.append(_section("quality_stat", "Quality statistics",
                      *[_curves(types[w], blocks[w], False, is_rna, blocks[w]["base_contents"]) for w in (0, 1)]))
    o.append(_section("contents_stat", "Base contents statistics",
                      *[_curves(types[w], blocks[w], True, is_rna, blocks[w]["base_contents"]) for w in (0, 1)]))
    o.append(_section("kmer_stat", "k-mer statistics", *[_kmer(types[w], blocks[w], is_rna) for w in (0, 1)]))
    o.append(f"\n</div>\n<div id='footer'> <p>{command}</p>fastplong {version}, at {time_text} </div></body></html>")
    return "".join(o).encode()
