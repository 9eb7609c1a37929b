#!/usr/bin/env python
"""Write the full SASS listing of every kernel in the built extension to <out>/<kernel>.sass
(cuobjdump -sass of the sm_90a objects, one file per entry point) plus an index with the mnemonics that show the
Hopper paths: HGMMA / WARPGROUP (wgmma), UTMALDG (TMA), SYNCS (mbarrier), LDGMC (multimem, NVLS).
Needs no GPU.  Usage: python scripts/dump_sass.py [out_dir]   (default: eventgrad_b200/csrc/build/sass)"""
import os, re, subprocess, sys, collections
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "eventgrad_b200", "csrc", "build")
KEY = ["HGMMA", "WARPGROUP", "UTMALDG", "SYNCS", "LDGMC", "REDG", "MEMBAR.SC.SYS", "ATOMS", "HMMA", "FFMA"]


def demangle(n):
    try:
        return subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip() or n
    except Exception:
        return n


def main():
    OUT = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else os.path.join(BUILD, "sass")
    os.makedirs(OUT, exist_ok=True)
    for f in os.listdir(OUT):
        os.remove(os.path.join(OUT, f))
    index = []
    for obj in sorted(os.listdir(BUILD)):
        if not obj.endswith(".cu.o"):
            continue
        txt = subprocess.run(["cuobjdump", "-sass", os.path.join(BUILD, obj)], capture_output=True, text=True).stdout
        parts = re.split(r"\n\s*Function : ", txt)
        for part in parts[1:]:
            name, _, body = part.partition("\n")
            name = name.strip()
            dm = demangle(name)
            short = re.sub(r"[^A-Za-z0-9_]+", "_", dm.split("(")[0].replace("egb::", "").replace("void ", ""))[:80].strip("_")
            path = os.path.join(OUT, f"{obj[:-5]}__{short}.sass")
            with open(path, "w") as fo:
                fo.write(f"// {dm}\n// object: csrc/build/{obj}  (nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3)\n")
                # drop the raw 128-bit encodings (hex comments): they triple the size and add nothing to a review
                lean = re.sub(r"[ \t]*/\* 0x[0-9a-f]{16} \*/", "", body)
                lean = "\n".join(l.rstrip() for l in lean.split("\n") if l.strip())
                fo.write("        Function : " + name + "\n" + lean + "\n")
            ops = collections.Counter(m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", body))
            n_ins = sum(ops.values())
            hits = {k: sum(v for o, v in ops.items() if o.startswith(k)) for k in KEY}
            index.append((os.path.basename(path), dm, n_ins, {k: v for k, v in hits.items() if v}))
    with open(os.path.join(OUT, "INDEX.md"), "w") as fo:
        fo.write("# SASS listings (cuobjdump -sass, sm_90a) -- one file per kernel entry point\n\n"
                 "| file | kernel | instructions | notable mnemonics |\n|---|---|---|---|\n")
        for f, dm, n, hits in index:
            fo.write(f"| `{f}` | `{dm[:110]}` | {n} | {', '.join(f'{k}x{v}' for k, v in hits.items())} |\n")
    print(f"wrote {len(index)} listings to {OUT}")


if __name__ == "__main__":
    main()
