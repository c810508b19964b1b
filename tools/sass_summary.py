"""Per-kernel SASS mnemonic census (proof of wgmma / TMA / multimem use), printed or written as markdown."""
import collections
import re
import subprocess
import sys

OBJS = ["gemm_sm90.cu.o", "attention_sm90.cu.o", "comm.cu.o", "elementwise.cu.o", "layernorm_stream.cu.o"]
INTEREST = re.compile(r"^(HGMMA|WARPGROUP|UTMALDG|UTMASTG|UBLKCP|SYNCS|MULTIMEM|"
                      r"LDGMC|LDG\.E\.NA|STG\.E\.NA|LDG\.E\.STRONG|STG\.E\.STRONG|LDG\.E\.128|STG\.E\.128|RED|ATOM|MEMBAR|HMMA|UCGABAR)")


def census(build_dir, objs=None):
    """{object file: {demangled kernel name: Counter(mnemonic -> count)}} for the mnemonics of interest."""
    out = collections.OrderedDict()
    for obj in objs or OBJS:
        txt = subprocess.run(["cuobjdump", "-sass", f"{build_dir}/{obj}"], capture_output=True, text=True).stdout
        mangled = re.findall(r"Function : (\S+)", txt)
        names = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True).stdout.split("\n")
        pretty = {}
        for m, n in zip(mangled, names):
            n = re.sub(r"\(anonymous namespace\)::", "", n.strip())
            pretty[m] = re.sub(r"\(.*", "", n)
        fn, counts = None, collections.OrderedDict()
        for ln in txt.splitlines():
            m = re.search(r"Function : (\S+)", ln)
            if m:
                fn = pretty[m.group(1)]
                counts[fn] = collections.Counter()
                continue
            m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Z][A-Z0-9_.]*)", ln)
            if m and fn:
                op = m.group(1)
                if INTEREST.match(op):
                    counts[fn][op] += 1
        out[obj] = counts
    return out


def main(build_dir, out):
    lines = ["# SASS census of the hand-written kernels (cuobjdump -sass, sm_90a)", "",
             "`HGMMA` = wgmma.mma_async, `WARPGROUP.*` = wgmma fence / commit / wait, `UTMALDG/UTMASTG` = TMA tensor "
             "load/store, `SYNCS.*` = mbarrier, `LDGMC...F32ADD` = multimem.ld_reduce (NVLS in-switch reduce), "
             "`LDG.E.NA.128` = streaming peer loads, `*.STRONG.SYS` = cross-GPU flags.", ""]
    for obj, counts in census(build_dir).items():
        lines.append(f"## {obj}")
        lines.append("")
        for fn, c in counts.items():
            if not c:
                continue
            lines.append(f"* `{fn[:150]}`: " + ", ".join(f"{k}×{v}" for k, v in sorted(c.items())))
        lines.append("")
    open(out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines[:40]))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "vit_10b_fsdp_example_b200/csrc/build",
         sys.argv[2] if len(sys.argv) > 2 else "sass_summary.md")
