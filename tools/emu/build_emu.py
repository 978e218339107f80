"""Prepare host-compilable copies of the HashAgg kernel sources for the thread-per-lane emulator (tools/emu):
copies blaze_b200/csrc/{vm.h,vm.cuh,kernels.cuh,kernels_fast.cuh,agg_device.cuh,kernels_fast.cu,kernels.cu} into <out>/, rewrites every
inline-PTX statement into the host helper of tools/emu/include/cuda_runtime.h, and rewrites every
`kernel<<<grid, block, smem, stream>>>(args)` into `emu::Launcher(grid, block, smem, stream).run(...)`, so that the
real launchers / dispatcher run too.  The product sources are not modified."""
import os, re, sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SRC = os.path.join(ROOT, "blaze_b200", "csrc")

ASM = re.compile(r'asm\s*(?:volatile)?\s*\(\s*"((?:[^"\\]|\\.)*)"\s*(.*?)\)\s*;', re.S)
LAUNCH = re.compile(r"([A-Za-z_]\w*(?:<[^<>;(){}]*>)?)<<<([^>]*)>>>\(([^;{}]*?)\)(?=\s*(?:;|\\|$|\}|else))", re.M)
OPERAND = re.compile(r'"[^"]*"\s*\(([^()]*(?:\([^()]*\)[^()]*)*)\)')


def translate(m):
    ptx, rest = m.group(1), m.group(2)
    parts = rest.split(":")
    outs = OPERAND.findall(parts[1]) if len(parts) > 1 else []
    ins = OPERAND.findall(parts[2]) if len(parts) > 2 else []
    op = ptx.split()[0]
    if ptx.startswith("{") and re.search(r"@\w+ ld\.global\.nc", ptx):          # `setp` + predicated load: (pointer, predicate, policy) -> "+" outputs
        return f"if ({ins[1]}) {{ " + " ".join(f"{o} = ({ins[0]})[{i}];" for i, o in enumerate(outs)) + " }"
    if "mbarrier" in ptx or "cp.async.bulk" in ptx or op.startswith("fence."): return ";"      # TMA staging: never reached on the emulated device (compiled out)
    if op == "ld.relaxed.gpu.global.u64": return f"{outs[0]} = emu_ld64({ins[0]});"
    if op == "ld.relaxed.gpu.global.v2.u64": return f"{outs[0]} = emu_ld64({ins[0]}); {outs[1]} = emu_ld64({ins[0]} + 1);"
    if op == "st.release.gpu.global.u32": return f"emu_st_release32({ins[0]}, {ins[1]});"
    if op == "st.relaxed.gpu.global.u64": return f"emu_st64({ins[0]}, {ins[1]});"
    if op == "red.global.add.u64": return f"emu_red_add_u64({ins[0]}, {ins[1]});"
    if op == "red.global.add.f64": return f"emu_red_add_f64({ins[0]}, {ins[1]});"
    if op == "red.global.min.s64": return f"emu_red_min_s64({ins[0]}, {ins[1]});"
    if op == "red.global.max.s64": return f"emu_red_max_s64({ins[0]}, {ins[1]});"
    if op == "mov.u32" and "lanemask_lt" in ptx: return f"{outs[0]} = emu_lanemask_lt();"
    if op.startswith("createpolicy"): return f"{outs[0]} = 0;"
    if op.startswith("ld.global.nc"):
        return " ".join(f"{o} = ({ins[0]})[{i}];" for i, o in enumerate(outs))
    raise SystemExit(f"build_emu: no host translation for PTX `{ptx}`")


def main(top):
    import shutil
    out = os.path.join(top, "blaze_b200", "csrc")              # same relative layout as the repo: sources include ../../include/blaze_b200.h
    os.makedirs(out, exist_ok=True)
    os.makedirs(os.path.join(top, "include"), exist_ok=True)
    shutil.copy(os.path.join(ROOT, "include", "blaze_b200.h"), os.path.join(top, "include", "blaze_b200.h"))
    for fn in sorted(f for f in os.listdir(SRC) if f.endswith((".h", ".cuh", ".cu", ".cc"))):
        s = open(os.path.join(SRC, fn)).read()
        s, n = ASM.subn(translate, s)
        s, nl = LAUNCH.subn(r"emu::Launcher(\2).run([&] { (\1)(\3); })", s)     # kernel<<<grid, block, smem, stream>>>(args)
        if "asm" in re.sub(r"//.*", "", s).replace("asm_", ""):
            left = [l for l in s.splitlines() if re.search(r"\basm\b", re.sub(r"//.*", "", l))]
            if left: raise SystemExit(f"build_emu: untranslated asm in {fn}: {left[:3]}")
        open(os.path.join(out, fn), "w").write(s)
        print(f"{fn}: {n} PTX statements translated, {nl} launches rewritten")


if __name__ == "__main__":
    main(sys.argv[1])
