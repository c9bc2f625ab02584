"""Static SASS instruction count per CUDA source line of one kernel (needs -lineinfo; no GPU).
usage: python tools/sass_lines.py <kernel-substring> [top]"""
import collections, os, re, subprocess, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "densesurfelmapping_b200", "libdsm_b200.so")
pat, top = sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 30
tmp = tempfile.mkdtemp()
subprocess.run(["cuobjdump", "-xelf", "all", lib], cwd=tmp, capture_output=True)
for cub in sorted(f for f in os.listdir(tmp) if f.endswith(".cubin")):  # the cubin that holds the kernel
    txt = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(tmp, cub)], capture_output=True, text=True).stdout.splitlines()
    if any(l.startswith(".text.") and pat in l for l in txt):
        break
src = {}  # source file named in the line info -> its lines
fn = cur = None
cnts = {}
for l in txt:
    m = re.match(r'\s*\.text\.(\S+):', l)
    if m:
        fn, cur = m.group(1), None
        cnts.setdefault(fn, collections.Counter())
        continue
    m = re.search(r'//## File ".*?([^/"]+)", line (\d+)', l)
    if m:
        cur = (m.group(1), int(m.group(2)))
        continue
    if fn and re.match(r'\s+/\*[0-9a-f]{4}\*/', l):
        cnts[fn][cur] += 1
for f, c in cnts.items():
    if pat in f:
        print(f, "total", sum(c.values()))
        for k, n in sorted(c.items(), key=lambda kv: -kv[1])[:top]:
            if k is None:
                print(f"{n:5d}  ?")
                continue
            fl, ln = k
            if fl not in src:
                path = os.path.join(ROOT, "densesurfelmapping_b200", "csrc", fl)
                src[fl] = open(path).read().splitlines() if os.path.exists(path) else []
            print(f"{n:5d}  {fl}:{ln}: {src[fl][ln - 1].strip()[:105] if ln <= len(src[fl]) else ''}")
