#!/usr/bin/env python
"""Static audit of the built libraries (no GPU needed): for the hot kernels of every variant, registers / shared
memory / spills from the ptxas log, the SASS instruction count, the mix by issue pipe and the mnemonics that
prove the bulk-copy (TMA) and mbarrier paths are what actually got compiled.

    python profiles/sass_audit.py > sass_audit.txt
"""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ntsc-crt_b200", "lib")

HOT = {  # variant -> substrings of the kernels worth listing
    "ntsc": ["k_mod_skeleton_rgb", "k_mod_picture_rgb_stagedILi5ELb1", "6k_syncE", "k_lines2ILi1ELi5", "k_lines2ILi0ELi5",
             "k_linesILb1ELi1ELi5", "k_linesILb0ELi1ELi5"],
    "ntsc_conv": ["k_lines_firILb1ELi1ELi5", "k_lines_firILb0ELi1ELi5"],
    "ntsc_conv4": ["k_lines_firILb1ELi1ELi5"],
    "vhs": ["k_noise_vhs", "6k_syncE"],
    "nes_p0": ["k_nes_table", "k_mod_nes"],
    "snes": ["k_mod_snes"],
    "nesrgb": ["k_mod_nesrgb"],
    "template": ["k_mod_skeleton_rgb", "k_mod_picture_rgb_stagedILi5ELb1", "6k_syncE"],
    "pv1k": ["k_mod_skeleton_rgb", "k_mod_picture_rgbEPK", "6k_syncE", "k_linesILb1ELi1ELi5", "k_linesILb0ELi1ELi5"],
    "ntsc_bloom": ["k_bloom", "k_lines_bloom"],
}

FMA = ("IMAD", "FFMA", "FMUL", "FADD", "HFMA2")
ALU = ("IADD3", "VIADD", "LOP3", "SHF", "LEA", "PRMT", "VIMNMX", "ISETP", "SEL", "IABS", "POPC", "FLO", "BREV", "I2I", "VABSDIFF", "PLOP3", "MOV", "CS2R")
LSU = ("LDS", "STS", "LDG", "STG", "LD", "ST", "LDGSTS", "ATOMS", "ATOMG", "RED", "LDC", "LDL", "STL", "SHFL", "MATCH", "VOTE")


def ptxas_info(variant):
    info = {}
    path = os.path.join(LIB, "build_%s.log" % variant)
    if not os.path.exists(path):
        return info
    cur = None
    for line in open(path, errors="replace"):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            info.setdefault(cur, {})["spill"] = int(m.group(2)) + int(m.group(3))
        m = re.search(r"Used (\d+) registers(?:, used \d+ barriers)?(?:, (\d+) bytes smem)?", line)
        if m and cur:
            info.setdefault(cur, {}).update(regs=int(m.group(1)), smem=int(m.group(2) or 0))
    return info


def sass_functions(variant):
    out = subprocess.run(["cuobjdump", "-sass", os.path.join(LIB, "libcrt_b200_%s.so" % variant)],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout.decode(errors="replace")
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur:
            ins = m.group(1).strip()
            ins = re.sub(r"^@!?U?P\d+\s+", "", ins)
            funcs[cur].append(ins.split()[0])
    return funcs


def main():
    for variant, wanted in HOT.items():
        if not os.path.exists(os.path.join(LIB, "libcrt_b200_%s.so" % variant)):
            continue
        info, funcs = ptxas_info(variant), sass_functions(variant)
        print("== libcrt_b200_%s.so" % variant)
        for want in wanted:
            for name, ops in funcs.items():
                if want not in name:
                    continue
                base = collections.Counter(o.split(".")[0] for o in ops)
                fma = sum(v for k, v in base.items() if k in FMA)
                alu = sum(v for k, v in base.items() if k in ALU)
                lsu = sum(v for k, v in base.items() if k in LSU)
                uni = sum(v for k, v in base.items() if k.startswith("U") and k not in ("UBLKCP",))
                i = info.get(name, {})
                print("  %s" % name)
                print("     registers %s  static smem %s B  spills %s B  SASS instructions %d" % (
                    i.get("regs", "?"), i.get("smem", "?"), i.get("spill", "?"), len(ops)))
                print("     by pipe: fma-side %d, alu-side %d, load/store %d, uniform datapath %d, other %d" % (
                    fma, alu, lsu, uni, len(ops) - fma - alu - lsu - uni))
                full = collections.Counter(ops)
                proof = {k: v for k, v in full.items() if k.startswith(("UBLKCP", "SYNCS", "UTMA", "LDGSTS", "FENCE", "VIMNMX.RELU"))}
                print("     bulk-copy / mbarrier / async evidence: %s" % (", ".join("%s x%d" % kv for kv in sorted(proof.items())) or "none"))
                print("     top opcodes: %s" % ", ".join("%s %d" % kv for kv in full.most_common(8)))


if __name__ == "__main__":
    main()
