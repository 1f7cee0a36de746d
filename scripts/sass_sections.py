"""Static size of the env-step path of one rollout-kernel variant, from its SASS and -lineinfo line tables.

    python scripts/sass_sections.py [--variant 1 | --shape go2] [--cubin FILE]

Compiles `dial_rollout_variant.cu` for the variant (or for the shape-specialised star<3,6> kernel of that
name, with the structure defines the library build uses) with the library's nvcc flags (or reads a cubin),
prints ptxas' register / stack / spill report, and attributes the SASS bytes of the kernel to source:
  * the cold tail (the divergent fall-backs of the warp shuffles that ptxas places after the last
    EXIT: taken only when a shuffle runs under a partial mask) is counted apart;
  * the env-step loop is every instruction inlined from rollout_warp's `for (int t ...)` loop, in the
    static-row copy of rollout_warp (the one every star and tree launch runs);
  * inside it, each byte goes to the physics_step phase it was inlined from (the `// ---- N.` headers),
    the Newton loop body (`while (!done)` of the star path) and the innermost source function.
The rollout kernel is bound by instruction delivery (DESIGN.md §5): the bytes streamed per env step,
and whether the Newton loop body fits the SM's instruction cache, are what its time follows."""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

HDR = "dial_device.cuh"
VAR = "dial_rollout_variant.cu"


def compile_cubin(variant, out, shape=None):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = [f"-DDIAL_VARIANT={variant}"]
    if shape:
        defs = dict(g._shape_defines())
        if shape not in defs:
            raise SystemExit(f"unknown shape {shape!r} (known: {', '.join(defs)})")
        flags = ["-DDIAL_VARIANT=1", f"-DDIAL_SHAPE_NAME={shape}"] + [f"-D{d}" for d in defs[shape]]
    cmd = [nvcc] + g.NVCC_FLAGS + flags + ["-Xptxas", "-v", "-cubin", "-o", out, os.path.join(g.CSRC, VAR)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(r.stderr)
    lines = r.stderr.splitlines()
    for i, l in enumerate(lines):
        if "Function properties for" in l and "rollout_kernel" in l:
            print("ptxas:", lines[i + 1].strip(), "|", lines[i + 2].split(":", 1)[1].strip())


def functions_of(lines):
    """Name of the enclosing DEV function for every line of the header (1-based)."""
    func_of, cur = {}, "?"
    for i, l in enumerate(lines, 1):
        if l.startswith("DEV ") and "(" in l:
            m = re.search(r"\b(\w+)\s*\(", l[4:])
            if m:
                cur = m.group(1)
        func_of[i] = cur
    return func_of


def block_span(lines, start):
    """Lines [start, end] of the brace block that opens on line `start` (1-based)."""
    depth = 0
    for i in range(start, len(lines) + 1):
        code = lines[i - 1].split("//")[0]
        depth += code.count("{") - code.count("}")
        if depth == 0 and i > start:
            return start, i
    raise SystemExit(f"no end of the block at {HDR}:{start}")


def find_line(lines, func_of, func, pattern, after=0):
    for i, l in enumerate(lines, 1):
        if i > after and func_of[i] == func and re.search(pattern, l):
            return i
    raise SystemExit(f"{pattern!r} not found in {func}")


def parse_sass(dis):
    """[(address, text, chain)] of the kernel; chain = [(file, line)] innermost first."""
    out, chain, in_group = [], [], False
    for l in dis.splitlines():
        s = l.strip()
        if s.startswith("//## File"):
            file, line = re.findall(r'"([^"]+)", line (\d+)', s)[0]
            if not in_group:
                chain, in_group = [], True
            chain.append((os.path.basename(file), int(line)))
            continue
        m = re.match(r"^/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;?$", s)
        if m:
            in_group = False
            out.append((int(m.group(1), 16), m.group(2), chain))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", type=int, default=1)
    ap.add_argument("--shape", help="the shape-specialised star<3,6> kernel of this name (e.g. go2)")
    ap.add_argument("--cubin", help="read this cubin instead of compiling the variant (it must be built with -lineinfo)")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        cubin = args.cubin
        if not cubin:
            cubin = os.path.join(tmp, f"rollout_{args.shape or 'v%d' % args.variant}.cubin")
            compile_cubin(args.variant, cubin, args.shape)
        dis = subprocess.run([os.environ.get("NVDISASM", "/usr/local/cuda/bin/nvdisasm"), "-gi", "-c", cubin],
                             capture_output=True, text=True, check=True).stdout
    insts = parse_sass(dis)
    hdr = open(os.path.join(g.CSRC, HDR)).read().splitlines()
    func_of = functions_of(hdr)
    t0, t1 = block_span(hdr, find_line(hdr, func_of, "rollout_warp", r"for \(int t = 0; t < H; \+\+t\) \{"))
    p9 = find_line(hdr, func_of, "physics_step", r"// ---- 9\. ")
    n0, n1 = block_span(hdr, find_line(hdr, func_of, "physics_step", r"while \(!done\) \{", after=p9))
    phase_of, cur = {}, "0. set-up"
    for i, l in enumerate(hdr, 1):
        m = re.match(r"\s*// ---- (\d+\..*?) -*$", l)
        if m and func_of[i] == "physics_step":
            cur = m.group(1).strip()
        phase_of[i] = cur

    last_exit = max(a for a, t, _ in insts if t == "EXIT")
    main_b = sum(16 for a, _, _ in insts if a <= last_exit)
    cold_b = 16 * len(insts) - main_b
    copies = sorted({ch[-1][1] for a, _, ch in insts if a <= last_exit and ch and ch[-1][0] == VAR
                     and any(f == HDR and func_of.get(n) == "rollout_warp" for f, n in ch)})
    static_row = copies[-1]   # the static-row call follows the dense path's persistent loop in the kernel source
    step_b, newton_b = 0, 0
    by_section, by_func = collections.Counter(), collections.Counter()
    for a, _, ch in insts:
        if a > last_exit or not ch or ch[-1] != (VAR, static_row):
            continue
        rw = next((n for f, n in ch if f == HDR and func_of.get(n) == "rollout_warp"), None)
        if rw is None or not (t0 <= rw <= t1):
            continue
        step_b += 16
        ps = next((n for f, n in reversed(ch) if f == HDR and func_of.get(n) == "physics_step"), None)
        if ps is None:
            section = f"rollout_warp: {hdr[rw - 1].strip()[:60]}"
        elif n0 <= ps <= n1:
            section = "9. Newton loop body"
            newton_b += 16
        else:
            section = "physics_step " + phase_of[ps]
        by_section[section] += 16
        f, n = ch[0] if ch else ("?", 0)
        by_func[func_of.get(n, "?") if f == HDR else f] += 16

    print(f"kernel: {16 * len(insts) / 1024:.1f} KB of SASS = {main_b / 1024:.1f} KB main body "
          f"+ {cold_b / 1024:.1f} KB cold tail (shuffle fall-backs after the last EXIT)")
    print(f"copies of rollout_warp: {len(copies)} (inlined at {VAR} lines {copies})")
    print(f"env-step loop ({HDR}:{t0}-{t1}) of the static-row copy ({VAR}:{static_row}): {step_b / 1024:.1f} KB")
    print(f"Newton loop body ({HDR}:{n0}-{n1}): {newton_b / 1024:.1f} KB")
    print("\n| section of the env-step loop | KB |\n|---|---|")
    for s, b in sorted(by_section.items(), key=lambda kv: -kv[1]):
        print(f"| {s} | {b / 1024:.1f} |")
    print("\n| innermost function (env-step loop) | KB |\n|---|---|")
    for s, b in by_func.most_common(20):
        print(f"| `{s}` | {b / 1024:.1f} |")


if __name__ == "__main__":
    main()
