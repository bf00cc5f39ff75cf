"""profiles/<tag>_sass_excerpts.md: per hot kernel, the SASS mnemonics that back the claims in DESIGN.md (packed
binary32 math, bulk / async copies, FP64 trig, shared-memory atomics; no tensor-core instructions on purpose).
Runs without a GPU: `cuobjdump -sass cpprobotics_b200/lib/libcrb.so`.   usage: python scripts/sass_excerpts.py r2"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tag = sys.argv[1] if len(sys.argv) > 1 else "r2"
so = os.path.join(ROOT, "cpprobotics_b200", "lib", "libcrb.so")
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
funcs = collections.OrderedDict()
cur = None
for line in txt.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        funcs[cur] = []
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4})\*/\s+(.*?);", line)
    if m and cur is not None:
        funcs[cur].append((m.group(1), m.group(2).strip()))
HOT = ["crb_ekf_step_kernel<128, 4, 2>", "crb_ekf_step_kernel<256, 3, 1>", "crb_pf_predict_weight_lean_kernel<128, 12>",
       "crb_mpc_tasks_kernel", "crb_mpc_solve_kernel<0>", "crb_lqr_dlqr_kernel<4, 1>", "crb_probe_ffma_kernel"]
WATCH = ["FFMA2", "FADD2", "FMUL2", "FFMA", "FMUL", "FADD", "DFMA", "DMUL", "DADD", "MUFU", "UBLKCP", "UTMALDG", "LDGSTS",
         "SYNCS", "LDG", "STG", "LDS", "STS", "ATOMS", "ATOMG", "NANOSLEEP", "SHFL", "VOTE", "HMMA", "UTCHMMA", "UTCQMMA", "BRA"]
out = [f"# {tag} — SASS evidence per hot kernel (`cuobjdump -sass cpprobotics_b200/lib/libcrb.so`, sm_90a)", "",
       "Counts are static instructions of the kernel.  `FFMA2/FADD2/FMUL2` = packed binary32 (two IEEE-rounded lanes per issue "
       "slot); `UBLKCP` = `cp.async.bulk` (TMA engine, 1-D); `LDGSTS` = `cp.async`; `SYNCS` = mbarrier; `DFMA/DMUL` = the "
       "binary64 sin/cos that carries the host libm's bits; `ATOMS` = shared-memory atomics (the task scheduler's lock).  "
       "`HMMA`/`UTC*MMA` (tensor cores) are absent on purpose: the work is 4x4 / 6x6 binary32 algebra that must match the "
       "reference's arithmetic, not a dense low-precision contraction.", ""]
for want in HOT:
    name = next((k for k in funcs if k.endswith(want) or want in k), None)
    if name is None:
        continue
    ins = funcs[name]
    c = collections.Counter(re.sub(r"^@!?U?P\d+\s+", "", t).split()[0].split(".")[0] for _, t in ins)
    out += [f"## `{name}` — {len(ins)} instructions", "",
            "| " + " | ".join(k for k in WATCH if c.get(k)) + " |", "|" + "---|" * sum(1 for k in WATCH if c.get(k)),
            "| " + " | ".join(str(c[k]) for k in WATCH if c.get(k)) + " |", "", "```"]
    shown = set()
    for key in ("FFMA2", "UBLKCP", "LDGSTS", "DFMA", "ATOMS.CAS", "SYNCS", "NANOSLEEP", "LDG.E.128", "STG.E.128", "LDS.128"):
        for a, t in ins:
            if key in t and key not in shown:
                out.append(f"/*{a}*/  {t}")
                shown.add(key)
                break
    out += ["```", ""]
open(os.path.join(ROOT, "profiles", f"{tag}_sass_excerpts.md"), "w").write("\n".join(out))
print("\n".join(out[:60]))
