#!/bin/bash
# Register spills of the hot kernel, on the CPU (no GPU needed): compiles fastp_b200/csrc/fp_api.cu to a cubin with the flags of
# __graft_entry__.build() and prints
#   * the ptxas stack / spill figures of the PE and SE fp_chain2_kernel<PAIRED> and of their out-of-line callees,
#   * the local-memory loads / stores (LDL / STL) per source line of both kernels with their callees;
#     "loop" counts the ones inside a loop of the machine code (between a backward branch and its target).
# Usage: scripts/spill_report.sh [arch, default sm_90a] [nvcc flags ...]     e.g.  scripts/spill_report.sh sm_100a
set -euo pipefail
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
ARCH="${1:-sm_90a}"; shift || true
NVCC="${NVCC:-$(command -v nvcc || echo /usr/local/cuda/bin/nvcc)}"
NVDISASM="$(dirname "$NVCC")/nvdisasm"
TMP="$(mktemp -d)"; trap 'rm -rf "$TMP"' EXIT
"$NVCC" -gencode "arch=compute_${ARCH#sm_},code=$ARCH" -O3 -lineinfo -std=c++17 --fmad=false -Xptxas -v "$@" \
    -I "$ROOT/include" -I "$ROOT/fastp_b200/csrc" -cubin "$ROOT/fastp_b200/csrc/fp_api.cu" -o "$TMP/k.cubin" 2> "$TMP/ptxas.txt"
"$NVDISASM" --print-line-info -c "$TMP/k.cubin" > "$TMP/k.sass"
python3 - "$TMP/ptxas.txt" "$TMP/k.sass" "$ARCH" <<'PY'
import collections, re, subprocess, sys
ptxas, sass, arch = sys.argv[1:4]

def demangle(names):
    try:
        out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
        return dict(zip(names, out))
    except (OSError, subprocess.CalledProcessError):
        return {n: n for n in names}

# ptxas -v: "Compiling entry function 'K'" opens a kernel; "Function properties for F" + the next line give F's frame and spills
print(f"== ptxas, {arch}: stack frame / spill stores / spill loads (bytes per thread); callees listed under the kernel they follow")
kernel, prop, rows = None, None, []
for line in open(ptxas):
    m = re.search(r"Compiling entry function '(\S+)'", line)
    if m: kernel = m.group(1) if "fp_chain2_kernel" in m.group(1) else None; continue
    m = re.search(r"Function properties for (\S+)", line)
    if m: prop = m.group(1); continue
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
    if m and prop and kernel:
        rows.append((kernel, prop, *map(int, m.groups())))
    prop = None
    m = re.search(r"Used (\d+) registers", line)
    if m and kernel: rows.append((kernel, "registers", int(m.group(1)), 0, 0))
dm = demangle(sorted({r[0] for r in rows} | {r[1] for r in rows}))
for k in sorted({r[0] for r in rows}, key=lambda k: dm[k]):
    own = [r for r in rows if r[0] == k]
    reg = [r[2] for r in own if r[1] == "registers"]
    for r in own:
        if r[1] == k: print(f"{dm[k].split('(')[0]:<40} {r[2]:5d} / {r[3]:5d} / {r[4]:5d}   {reg[0] if reg else '?'} registers")
    for r in own:
        if r[1] not in (k, "registers") and (r[3] or r[4]): print(f"    {dm[r[1]].split('(')[0]:<36} {r[2]:5d} / {r[3]:5d} / {r[4]:5d}")

# SASS: per function (the kernel and its out-of-line callees, named "$kernel$callee"), LDL / STL by the source line above them
funcs = collections.OrderedDict()
cur, line_of = None, "?"
for ln in open(sass):
    m = re.match(r"\s*\.text\.(\S+):", ln) or re.match(r"(\$\S+\$\S+):", ln)
    if m: cur = m.group(1); funcs[cur] = {"ins": [], "labels": {}}; line_of = "?"; continue
    if cur is None: continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
    if m: line_of = f"{m.group(1).split('/')[-1]}:{m.group(2)}"; continue
    m = re.match(r"(\.L_x_\d+):", ln.strip())
    if m: funcs[cur]["labels"][m.group(1)] = len(funcs[cur]["ins"]); continue
    m = re.match(r"\s*/\*([0-9a-f]+)\*/\s+(.*?);", ln)
    if m: funcs[cur]["ins"].append((line_of, m.group(2)))
for want in ("_Z16fp_chain2_kernelILb1EEv14fp_launch_args", "_Z16fp_chain2_kernelILb0EEv14fp_launch_args"):
    mine = [f for f in funcs if f == want or f.startswith("$" + want + "$")]
    per, tot = collections.Counter(), collections.Counter()
    for f in mine:
        ins, labels = funcs[f]["ins"], funcs[f]["labels"]
        loops = []                                   # [target, branch] index ranges of backward branches
        for i, (_, op) in enumerate(ins):
            m = re.search(r"\bBRA\b.*`\((\.L_x_\d+)\)", op)
            if m and m.group(1) in labels and labels[m.group(1)] <= i: loops.append((labels[m.group(1)], i))
        name = dm.get(f.split("$")[-1], None) if f != want else "[kernel body]"
        name = (name or demangle([f.split("$")[-1]])[f.split("$")[-1]]).split("(")[0]
        for i, (src, op) in enumerate(ins):
            kind = "LDL" if re.match(r"(@!?U?P\d\s+)?LDL\b", op) else "STL" if re.match(r"(@!?U?P\d\s+)?STL\b", op) else None
            if not kind: continue
            inloop = any(a <= i <= b for a, b in loops)
            per[(name, src, kind, inloop)] += 1; tot[kind] += 1; tot[kind + " in loops"] += inloop
    print(f"\n== {dm.get(want, want).split('(')[0]}, {arch}: LDL {tot['LDL']} ({tot['LDL in loops']} in loops), STL {tot['STL']} ({tot['STL in loops']} in loops)")
    keyed = collections.defaultdict(lambda: [0, 0, 0, 0])
    for (name, src, kind, inloop), n in per.items():
        k = keyed[(name, src)]; k[(0 if kind == "LDL" else 2) + (1 if inloop else 0)] += n
    print(f"  {'function':<28} {'source line':<22} {'LDL':>5} {'loop':>5} {'STL':>5} {'loop':>5}")
    for (name, src), v in sorted(keyed.items(), key=lambda kv: (kv[0][0] != "[kernel body]", kv[0][0], int(kv[0][1].split(":")[-1]) if kv[0][1][-1].isdigit() else 0)):
        print(f"  {name[:28]:<28} {src:<22} {v[0] + v[1]:5d} {v[1]:5d} {v[2] + v[3]:5d} {v[3]:5d}")
PY
