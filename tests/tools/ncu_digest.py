"""Digest of an ncu report: the launch's key raw metrics, stall reasons per issued instruction, and the
source lines (CUDA view, needs -lineinfo + --import-source on) that carry most stall samples / instructions.
  python tests/tools/ncu_digest.py report.ncu-rep [out.txt]      (runs `ncu -i`, so it works on the GPU box, where a
report of the big kernels is too large to bring back)"""
import collections
import csv
import io
import os
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__average_warp_latency_per_inst_issued.ratio", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "lts__t_bytes.sum", "l1tex__t_bytes.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__inst_executed_pipe_fp64.sum", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
        "smsp__sass_thread_inst_executed_op_dadd_pred_on.sum", "smsp__sass_thread_inst_executed_op_dmul_pred_on.sum",
        "smsp__sass_thread_inst_executed_op_dfma_pred_on.sum", "local_load_bytes", "smsp__inst_executed_op_local_ld.sum",
        "smsp__inst_executed_op_local_st.sum"]


def ncu(args):
    return subprocess.run(["ncu"] + args, capture_output=True, text=True).stdout


def main():
    rep = sys.argv[1]
    out = open(sys.argv[2], "w") if len(sys.argv) > 2 else sys.stdout
    raw = list(csv.reader(io.StringIO(ncu(["-i", rep, "--page", "raw", "--csv"]))))
    hdr = raw[0]
    for r in raw[2:]:
        d = dict(zip(hdr, r))
        out.write("== %s\n" % d.get("Kernel Name", "?")[:150])
        for k in KEYS:
            if k in d:
                out.write("  %-62s %s\n" % (k, d[k]))
        stalls = sorted(((float(v), k) for k, v in d.items() if k.startswith("smsp__average_warps_issue_stalled_")
                         and k.endswith("_per_issue_active.ratio") and v not in ("", "n/a")), reverse=True)
        out.write("  stall cycles per issued instruction: " + ", ".join(
            "%s %.2f" % (k[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")], v) for v, k in stalls[:9]) + "\n")
    src = ncu(["-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"])
    per = collections.defaultdict(lambda: [0, 0, 0])
    text = {}
    cur, hd = None, None
    for r in csv.reader(io.StringIO(src)):
        if not r:
            continue
        if r[0] == "Kernel Name":
            continue
        if r[0] == "File Path":
            cur = os.path.basename(r[1])
            continue
        if r[0] == "Function Name":
            continue
        if r[0] == "Line No":
            hd = r
            ii, it, isamp = hd.index("Instructions Executed"), hd.index("Thread Instructions Executed"), hd.index("# Samples")
            continue
        if r[0] != "" and hd:
            try:
                key = (cur, int(r[0]))
                per[key][0] += int(r[ii])
                per[key][1] += int(r[it])
                per[key][2] += int(r[isamp])
                text[key] = r[1].strip()[:100]
            except ValueError:
                pass
    tot = [sum(v[k] for v in per.values()) or 1 for k in range(3)]
    out.write("source view (all launches of the report): %d warp instructions, %.1f lanes per instruction, %d stall samples\n"
              % (tot[0], tot[1] / tot[0], tot[2]))
    byfile = collections.defaultdict(lambda: [0, 0, 0])
    for (fl, _), v in per.items():
        for k in range(3):
            byfile[fl][k] += v[k]
    for fl, v in sorted(byfile.items(), key=lambda x: -x[1][2]):
        out.write("  %-28s instructions %5.1f%%  lanes %5.1f  samples %5.1f%%\n" % (fl, 100 * v[0] / tot[0], v[1] / max(v[0], 1), 100 * v[2] / tot[2]))
    out.write("lines with the most stall samples:\n")
    for (fl, l), v in sorted(per.items(), key=lambda x: -x[1][2])[:40]:
        out.write("  %-18s %5d  samples %4.1f%%  instructions %4.1f%%  lanes %4.1f | %s\n"
                  % (fl, l, 100 * v[2] / tot[2], 100 * v[0] / tot[0], v[1] / max(v[0], 1), text[(fl, l)]))
    out.write("lines with the most executed instructions:\n")
    for (fl, l), v in sorted(per.items(), key=lambda x: -x[1][0])[:25]:
        out.write("  %-18s %5d  instructions %4.1f%%  lanes %4.1f  samples %4.1f%% | %s\n"
                  % (fl, l, 100 * v[0] / tot[0], v[1] / max(v[0], 1), 100 * v[2] / tot[2], text[(fl, l)]))


if __name__ == "__main__":
    main()
