"""SASS size of the tracker sweep: the instructions track_cluster_kernel issues per point evaluation (CPU only, not a test).

usage: python tests/_sass_track_sweep.py [lib.so | kernels.o] [--hist] [--list]

For every instantiation of track_cluster_kernel the script finds the sweep loop: the back-edge loop that contains the per-thread tap gathers
(LDGSTS, twelve per point) and no FP64 or shuffle instruction.  It reports
  * the loop's size, the points it evaluates per trip (LDGSTS / 12) and its local-memory (spill) instructions,
  * its steady path: the loop without the innermost forward-branch regions that hold the elected thread's chunk issue (UBLKCP, SYNCS.ARRIVE) or a
    division slow-path CALL, and without the chunk barrier and the wait for the next chunk (BAR.SYNC up to SYNCS.PHASECHK), i.e. what a warp issues
    per trip for points that take none of these (once per chunk, or rarely), and that per point,
  * with --hist, an opcode histogram of the steady path; with --list, the steady path itself.
"""
import os
import re
import shutil
import subprocess
import sys
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
if not os.path.exists(CUOBJDUMP):
    CUOBJDUMP = shutil.which("cuobjdump") or CUOBJDUMP
TAPS = 12
_FUNC = re.compile(r"Function : (\S+)")
_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
_KERN = re.compile(r"track_cluster_kernelILi(\d+)ELi(\d+)E")
# forward-branch regions that are not part of a steady point evaluation: the elected thread's chunk issue and the division slow paths
_COLD = re.compile(r"^(UBLKCP|SYNCS\.ARRIVE|CALL\.)")
_NOT_SWEEP = re.compile(r"^(DADD|DMUL|DFMA|SHFL)")


class Insn:
    __slots__ = ("addr", "pred", "op", "args", "text")

    def __init__(self, addr, text):
        self.addr, self.text = addr, text
        parts = text.split(None, 1)
        self.pred = parts[0] if parts[0].startswith("@") else None
        rest = text[len(parts[0]):].strip() if self.pred else text
        bits = rest.split(None, 1)
        self.op, self.args = bits[0], (bits[1] if len(bits) > 1 else "")

    @property
    def target(self):
        if not self.op.startswith("BRA"):
            return None
        m = re.search(r"(0x[0-9a-f]+)\s*$", self.args)
        return int(m.group(1), 16) if m else None


def functions(path):
    """{mangled name: [Insn]} of every function in the SASS of `path`."""
    out = subprocess.run([CUOBJDUMP, "-sass", path], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = _FUNC.search(line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = _INSN.search(line)
        if m and cur is not None:
            cur.append(Insn(int(m.group(1), 16), m.group(2)))
    return funcs


def sweep_loops(insns):
    """Back-edge loops [head, back-edge] that contain an LDGSTS and no FP64 or shuffle instruction (those belong to the block reduction and the LM control
    step of the loop around the sweep), as (first index, last index)."""
    idx = {ins.addr: i for i, ins in enumerate(insns)}
    loops = []
    for i, ins in enumerate(insns):
        t = ins.target
        if t is not None and t <= ins.addr and t in idx:
            body = insns[idx[t]:i + 1]
            if any(x.op.startswith("LDGSTS") for x in body) and not any(_NOT_SWEEP.match(x.op) for x in body):
                loops.append((idx[t], i))
    return loops


def cold_regions(insns, lo, hi):
    """For every cold instruction in [lo, hi], the innermost forward-branch region (the instructions a branch skips) around it; the union as index ranges."""
    idx = {ins.addr: i for i, ins in enumerate(insns)}
    regs = []
    for i in range(lo, hi + 1):
        t = insns[i].target
        if t is not None and t > insns[i].addr and t in idx and idx[t] <= hi + 1:
            regs.append((i + 1, idx[t] - 1))
    cold = set()
    for j in range(lo, hi + 1):
        if _COLD.match(insns[j].op):
            around = [r for r in regs if r[0] <= j <= r[1]]
            if around:
                a, b = min(around, key=lambda r: r[1] - r[0])
                cold.update(range(a, b + 1))
    for j in range(lo, hi + 1):                             # the chunk barrier and the wait for the next chunk: BAR.SYNC up to the mbarrier test and its retry branch
        if insns[j].op.startswith("BAR.SYNC"):
            e = j
            while e < hi and not insns[e].op.startswith("SYNCS.PHASECHK"):
                e += 1
            if e < hi and insns[e + 1].op.startswith("BRA"):
                e += 1
            cold.update(range(j, e + 1))
    out, run = [], None
    for j in sorted(cold):
        if run and j == run[1] + 1:
            run[1] = j
        else:
            run = [j, j]; out.append(run)
    return [tuple(r) for r in out]


def analyse(insns):
    loops = sweep_loops(insns)
    res = []
    for lo, hi in loops:
        cold = cold_regions(insns, lo, hi)
        skip = set()
        for a, b in cold:
            skip.update(range(a, b + 1))
        steady = [insns[i] for i in range(lo, hi + 1) if i not in skip]
        body = insns[lo:hi + 1]
        ldgsts = sum(x.op.startswith("LDGSTS") for x in body)
        local = sum(x.op.startswith(("LDL", "STL")) for x in body)
        res.append(dict(lo=body[0].addr, hi=body[-1].addr, size=len(body), ldgsts=ldgsts, points=ldgsts / TAPS, local=local,
                        steady=len(steady), steady_per_point=len(steady) / max(ldgsts / TAPS, 1e-9),
                        cold=[(insns[a].addr, insns[b].addr, b - a + 1) for a, b in cold],
                        hist=Counter(x.op.split(".")[0] for x in steady), steady_insns=steady))
    return res


def kernels(path):
    """{(THREADS, MINB): analyse(...)} for every track_cluster_kernel instantiation in `path`."""
    out = {}
    for name, insns in functions(path).items():
        m = _KERN.search(name)
        if m:
            out[(int(m.group(1)), int(m.group(2)))] = analyse(insns)
    return out


def main(argv):
    args = [a for a in argv if not a.startswith("--")]
    path = args[0] if args else os.path.join(ROOT, "sdv-loam_b200", "libsdv_b200.so")
    print(f"{path}")
    for (t, mb), loops in sorted(kernels(path).items()):
        print(f"track_cluster_kernel<{t},{mb}>: {len(loops)} sweep loop(s)")
        for L in loops:
            print(f"  loop 0x{L['lo']:x}-0x{L['hi']:x}: {L['size']} instructions, {L['ldgsts']} LDGSTS ({L['points']:g} point(s) per trip), {L['local']} local-memory (spill) instructions; "
                  f"steady path {L['steady']} = {L['steady_per_point']:.1f} per point; cold regions {[(hex(a), hex(b), n) for a, b, n in L['cold']]}")
            if "--hist" in argv:
                print("   ", ", ".join(f"{op} {n}" for op, n in L["hist"].most_common()))
            if "--list" in argv:
                for x in L["steady_insns"]:
                    print(f"    {x.addr:6x}  {x.text}")


if __name__ == "__main__":
    main(sys.argv[1:])
