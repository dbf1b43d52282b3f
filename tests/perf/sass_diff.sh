#!/bin/bash
# sass_diff.sh OLD.so NEW.so - do two builds of libsqllm_b200.so hold the same device code?
#
# Splits `cuobjdump -sass` of each library by function, drops addresses and instruction encodings, demangles the names and strips
# the anonymous-namespace qualifier (its mangled tag names the translation unit, so it differs when a kernel moves to another unit),
# then matches the kernels by that name.  Every kernel of OLD must appear in NEW with the same instructions and the same
# registers, stack, shared and local memory (`cuobjdump -res-usage`), and NEW may have no kernel that OLD lacks.  Needs no GPU.
# Prints one line per difference and a summary; exits 1 if anything differs.
set -euo pipefail
[ $# -eq 2 ] || { echo "usage: $0 OLD.so NEW.so" >&2; exit 2; }
filt=$(command -v cu++filt || echo /usr/local/cuda/bin/cu++filt)
dump() {  # $1 = library, $2 = sass | res-usage: demangled text without the anonymous-namespace qualifier
    cuobjdump -"$2" "$1" | "$filt" | sed -e 's/(anonymous namespace):://g' -e 's/<unnamed>:://g'
}
python3 - <(dump "$1" sass) <(dump "$2" sass) <(dump "$1" res-usage) <(dump "$2" res-usage) <<'EOF'
import collections, re, sys

def sass(path):  # function name -> list of SASS bodies (a name may occur once per translation unit)
    out, name = collections.defaultdict(list), None
    for line in open(path):
        m = re.match(r"\s*Function : (.*)$", line)
        if m:
            name = m.group(1).strip()
            out[name].append([])
        elif name and line.strip().startswith("/*") and re.match(r"\s*/\*[0-9a-f]{4,}\*/", line):
            ins = re.sub(r"/\*[0-9a-f]+\*/", "", line)
            ins = re.sub(r"/\* 0x[0-9a-f]+ \*/", "", ins)
            out[name][-1].append(" ".join(ins.split()))
    return out

def res(path):  # function name -> list of (REG, STACK, SHARED, LOCAL)
    out, name = collections.defaultdict(list), None
    for line in open(path):
        m = re.match(r"\s*Function (.*):\s*$", line)
        if m:
            name = m.group(1).strip()
            continue
        if name and "REG:" in line:
            f = dict(kv.split(":", 1) for kv in line.split())
            out[name].append(tuple(f[k] for k in ("REG", "STACK", "SHARED", "LOCAL")))
            name = None
    return out

old, new, rold, rnew = sass(sys.argv[1]), sass(sys.argv[2]), res(sys.argv[3]), res(sys.argv[4])
bad = 0
for k in sorted(set(old) | set(new)):
    a, b = old.get(k, []), new.get(k, [])
    if len(a) != len(b):
        print(f"COUNT  {k}: {len(a)} in OLD, {len(b)} in NEW")
        bad += 1
    elif sorted(a) != sorted(b):
        print(f"SASS   {k}")
        bad += 1
    elif sorted(rold.get(k, [])) != sorted(rnew.get(k, [])):
        print(f"USAGE  {k}: REG/STACK/SHARED/LOCAL {rold.get(k)} -> {rnew.get(k)}")
        bad += 1
n_old, n_new = sum(map(len, old.values())), sum(map(len, new.values()))
print(f"{n_old} kernels in OLD, {n_new} in NEW; {bad} differ" + ("" if bad else ": identical SASS and resource usage"))
sys.exit(1 if bad or not n_old else 0)
EOF
