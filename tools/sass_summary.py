"""Per kernel, how often the SASS mnemonics that prove (or disprove) a Hopper-native kernel occur — HGMMA / WARPGROUP
(wgmma), UTMALDG / UBLKCP / UBLKPF (TMA), HMMA (mma.sync), LDGSTS (cp.async), MUFU.EX2 — from `cuobjdump -sass` of the
objects libclengine.so is linked from.

    python tools/sass_summary.py [sass_summary.txt]
"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
OBJ = ROOT / "crowdllama_b200" / "lib" / "obj"
PAT = ["HGMMA", "WARPGROUP", "UTMALDG", "UBLKCP", "UBLKPF", "HMMA", "LDGSTS", "MUFU.EX2", "SYNCS", "LDSM"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return [re.sub(r"\(.*", "", n.replace("(anonymous namespace)::", "")).replace("void ", "").replace("cl::", "") for n in out]


def main(dst):
    lines = ["# SASS mnemonic counts per kernel (cuobjdump -sass of crowdllama_b200/lib/obj/*.o, sm_90a); 0 = absent; kernels without any",
             "# of these mnemonics are omitted",
             "# " + " ".join(f"{p:>8s}" for p in PAT) + "  kernel  [object]"]
    for obj in sorted(OBJ.glob("*.cu.o")):
        sass = subprocess.run(["cuobjdump", "-sass", str(obj)], capture_output=True, text=True).stdout
        cur, counts = None, collections.OrderedDict()
        for ln in sass.splitlines():
            m = re.search(r"Function : (\S+)", ln)
            if m:
                cur = m.group(1)
                counts[cur] = collections.Counter()
                continue
            if cur is None:
                continue
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?);", ln)
            if m:
                ins = m.group(1)
                for p in PAT:
                    if re.search(r"(^|\s)" + re.escape(p) + r"[A-Za-z0-9_.]*\s", ins + " "):
                        counts[cur][p] += 1
        names = demangle(list(counts))
        for (mangled, c), name in zip(counts.items(), names):
            if not sum(c.values()):
                continue
            lines.append("  " + " ".join(f"{c[p]:8d}" for p in PAT) + f"  {name[:90]}  [{obj.name}]")
    Path(dst).write_text("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else str(ROOT / "profiles" / "sass_summary.txt"))
