"""Static instruction counts of the primitive GJK passes, by phase (no GPU needed).

Compiles csrc/hfb_gjkpass.cu for sm_90a with the library's flags and -lineinfo, disassembles it with the inlined
line table (`nvdisasm -gi`) and attributes every SASS instruction of k_gjk_first<MODE, false> and
k_gjk_more<MODE, false> to a phase by the source frames it was inlined through:

  set-up        what runs once per pair before the iterations (pair inputs, Minkowski set-up, gjk_begin, pose rows)
  loop          the pass's own iteration loop around gjk_step
  step: ...     gjk_step, split at its comments (support direction and support call, check B, check C) and its
                simplex sub-solve by rank (1: the point, 2: project_line, 3: project_triangle, 4: project_tetra);
                "ray formula" is the segment or triangle ray the projections leave to the step; "rl, status" is
                the norm of the new ray and the status update after the sub-solve
  save / load   save_running, load_running, append_running
  finish_pair   the status machine, the witness points and the result record or EPA item of a finished pair
  fn <name>     an out-of-line function (prim_support, the projections of the witness points, the FP64 division
                and square-root slow paths)

For each phase it counts the instructions, the FP64 ones (DFMA, DMUL, DADD and the rest: DSETP, DMNMX, ...), MUFU,
branches (BRA, BSSY, BSYNC, CALL, RET, EXIT, ...), local-memory accesses (LDL / STL) and the calls into the division
(`div_rn_f64`) and square-root (`dsqrt_rn_f64`) slow paths.  The counts are static: an instruction counts once
however often it runs.

    python tests/tools/gjk_iter_sass.py [--mode 0|1] [--csrc DIR] [--keep DIR]
"""
import argparse
import collections
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..")
sys.path.insert(0, os.path.join(ROOT, "hpp-fcl_b200"))
import build as B  # noqa: E402  (the library's nvcc flags)

LINE_RE = re.compile(r'//## File "([^"]+)", line (\d+)')
INSN_RE = re.compile(r"/\*[0-9a-f]{4,}\*/\s+(@!?U?P[0-9T]+\s+)?([A-Z][A-Z0-9_.]*)(.*?);")
FUNC_RE = re.compile(r"^\s*\.type\s+(\S+),@function")
COLS = ["insns", "DFMA", "DMUL", "DADD", "FP64 other", "MUFU", "branch", "LDL/STL", "div slow", "sqrt slow"]
BRANCH = ("BRA", "BRX", "BSSY", "BSYNC", "CALL", "RET", "EXIT", "JMP", "JMX", "WARPSYNC", "BREAK")


def nvcc_cubin(csrc, out):
    flags = [f for f in B.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC", "-Xptxas", "-v")]
    cmd = [B._nvcc()] + flags + ["-I", os.path.join(csrc, "..", "..", "include"), "-I", csrc,
                                 "-cubin", "-o", out, os.path.join(csrc, "hfb_gjkpass.cu")]
    subprocess.run(cmd, check=True)
    nvdisasm = os.path.join(os.path.dirname(B._nvcc()), "nvdisasm")
    return subprocess.run([nvdisasm, "-gi", "-c", out], check=True, capture_output=True, text=True).stdout


def func_ranges(path, names):
    """{name: (first line, last line)} of the definitions of `names` in `path` (1-based; the body by brace count)"""
    lines = open(path).read().split("\n")
    out = {}
    for name in names:
        pat = re.compile(r"\b%s\s*\(" % re.escape(name))
        for k, ln in enumerate(lines):
            if pat.search(ln) and not ln.lstrip().startswith("//") and ";" not in ln.split("(")[0]:
                depth, seen, j = 0, False, k
                while j < len(lines):
                    code = lines[j].split("//")[0]
                    depth += code.count("{") - code.count("}")
                    seen = seen or "{" in code
                    if seen and depth == 0:
                        break
                    if not seen and ";" in code:  # a declaration or a call, not the definition
                        break
                    j += 1
                if seen and depth == 0:
                    out[name] = (k + 1, j + 1)
                    break
    return out


class Phases:
    def __init__(self, csrc):
        self.gjk = os.path.realpath(os.path.join(csrc, "hfb_gjk.cuh"))
        self.pass_ = os.path.realpath(os.path.join(csrc, "hfb_gjkpass.cu"))
        self.fr = func_ranges(self.gjk, ["gjk_step"])
        self.pr = func_ranges(self.pass_, ["save_running", "load_running", "append_running", "finish_pair",
                                           "k_gjk_first", "k_gjk_more"])
        lo, hi = self.fr["gjk_step"]
        src = open(self.gjk).read().split("\n")
        # gjk_step's segments, at its comments; the sub-solve by the line of each rank's branch
        marks = []
        for k in range(lo, hi):
            t = src[k - 1]
            for key, label in (("// support direction", "step: direction + support call"),
                               ("// check B", "step: check B"), ("// drop the momentum", "step: check B"),
                               ("// check C", "step: check C"), ("// simplex sub-solve", "step: sub-solve")):
                if key in t:
                    marks.append((k, label))
        self.marks = marks
        self.rank_line = {}
        for k in range(lo, hi):
            t = src[k - 1]
            if "g.ray = L.w" in t:
                self.rank_line[k] = "step: rank 1"
            for fn, r in (("project_line", 2), ("project_triangle", 3), ("project_tetra", 4)):
                if fn + "(g" in t:
                    self.rank_line[k] = "step: rank %d (%s)" % (r, fn)
            if "r.kind == RAY_" in t:
                self.rank_line[k] = "step: ray formula"
            if "L.rl = nrm(g.ray)" in t:
                self.rl_line = k

    def step_phase(self, line):
        label = "step: check A"
        for k, lab in self.marks:
            if line >= k:
                label = lab
        if label == "step: sub-solve":
            if line in self.rank_line:
                return self.rank_line[line]
            if line >= self.rl_line:
                return "step: rl, status"
        return label

    def of(self, frames, kernel):
        """frames: [(file, line)] innermost first"""
        def inside(f, l, path, rng):
            return f == path and rng[0] <= l <= rng[1]
        for f, l in frames:
            for fn in ("finish_pair",):
                if inside(f, l, self.pass_, self.pr[fn]):
                    return "finish_pair"
        for f, l in frames:
            for fn in ("save_running", "load_running", "append_running"):
                if inside(f, l, self.pass_, self.pr[fn]):
                    return "save / load"
        for f, l in frames:
            if inside(f, l, self.gjk, self.fr["gjk_step"]):
                return self.step_phase(l)
        f, l = frames[-1] if frames else ("", 0)
        if f == self.pass_ and kernel in self.pr and self.pr[kernel][0] <= l <= self.pr[kernel][1]:
            src_line = open(self.pass_).read().split("\n")[l - 1]
            if "gjk_step<" in src_line:
                return "loop"
        return "set-up"


def count(sass, csrc, kernels):
    ph = Phases(csrc)
    tables = {}
    cur_kernel, cur_func, frames, pending = None, None, [], []
    for raw in sass.split("\n"):
        if raw.startswith(".text."):
            name = raw[len(".text."):].rstrip(":")
            cur_kernel = next((k for k in kernels if k[1] in name), None)
            cur_func = None
            continue
        m = FUNC_RE.match(raw)
        if m and cur_kernel:
            nm = m.group(1)
            cur_func = None if "$" not in nm else nm.split("$")[-1]
            continue
        if cur_kernel is None:
            continue
        m = LINE_RE.search(raw)
        if m:
            pending.append((os.path.realpath(m.group(1)), int(m.group(2))))
            continue
        m = INSN_RE.search(raw)
        if not m:
            continue
        if pending:
            frames, pending = pending, []
        op, rest = m.group(2), m.group(3)
        if cur_func is None:
            phase = ph.of(frames, "k_gjk_first" if "first" in cur_kernel[0] else "k_gjk_more")
        else:
            short = re.sub(r"^__internal_\d+_", "", cur_func)
            short = re.sub(r"^_ZN3hfb\d+", "", short)
            short = re.sub(r"E.*$", "", short) if short.startswith(("prim", "proj")) else short
            phase = "fn " + short
        row = tables.setdefault(cur_kernel[0], collections.OrderedDict()).setdefault(phase, collections.Counter())
        row["insns"] += 1
        base = op.split(".")[0]
        if base in ("DFMA", "DMUL", "DADD"):
            row[base] += 1
        elif base.startswith("D") and base in ("DSETP", "DMNMX", "DSET"):
            row["FP64 other"] += 1
        if base == "MUFU":
            row["MUFU"] += 1
        if base in BRANCH:
            row["branch"] += 1
        if base in ("LDL", "STL"):
            row["LDL/STL"] += 1
        if base == "CALL" and "div_rn_f64" in rest:
            row["div slow"] += 1
        if base == "CALL" and "dsqrt_rn_f64" in rest:
            row["sqrt slow"] += 1
    return tables


ORDER = ["set-up", "loop", "step: check A", "step: direction + support call", "step: check B", "step: check C",
         "step: sub-solve", "step: rank 1", "step: rank 2 (project_line)", "step: rank 3 (project_triangle)",
         "step: rank 4 (project_tetra)", "step: ray formula", "step: rl, status", "save / load", "finish_pair"]


def render(tables):
    out = []
    for kname, rows in sorted(tables.items(), key=lambda kv: "more" in kv[0]):
        out.append("\n%s\n" % kname)
        out.append("| phase | " + " | ".join(COLS) + " |")
        out.append("|---" * (len(COLS) + 1) + "|")
        keys = [k for k in ORDER if k in rows] + sorted(k for k in rows if k not in ORDER)
        tot = collections.Counter()
        for k in keys:
            out.append("| %s | " % k + " | ".join(str(rows[k][c]) for c in COLS) + " |")
            if k.startswith("step: "):
                tot.update(rows[k])
        out.append("| gjk_step, inline total | " + " | ".join(str(tot[c]) for c in COLS) + " |")
    return "\n".join(out)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--mode", type=int, default=0, help="0: distance, 1: collide")
    ap.add_argument("--csrc", default=os.path.join(ROOT, "hpp-fcl_b200", "csrc"))
    ap.add_argument("--keep", default=None, help="also write the cubin and its disassembly to this directory")
    a = ap.parse_args()
    csrc = os.path.realpath(a.csrc)
    kernels = [("k_gjk_first<%d, false>" % a.mode, "k_gjk_firstILi%dELb0EE" % a.mode),
               ("k_gjk_more<%d, false>" % a.mode, "k_gjk_moreILi%dELb0EE" % a.mode)]
    tmp = tempfile.mkdtemp(prefix="gjk_iter_sass_")
    try:
        cubin = os.path.join(tmp, "hfb_gjkpass.cubin")
        sass = nvcc_cubin(csrc, cubin)
        if a.keep:
            os.makedirs(a.keep, exist_ok=True)
            shutil.copy(cubin, a.keep)
            with open(os.path.join(a.keep, "hfb_gjkpass.sass"), "w") as f:
                f.write(sass)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(render(count(sass, csrc, kernels)))


if __name__ == "__main__":
    main()
