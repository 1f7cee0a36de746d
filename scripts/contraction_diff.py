"""Where the fp32 rounding of the shape-specialised star<3,6> rollout kernel can part from the generic one's.

    python scripts/contraction_diff.py [--shape go2] [--all]

ShapeFixed (csrc/dial_device.cuh) turns warp-uniform counts into compile-time constants.  The arithmetic of
each row stays the same, but with other trip counts and fewer branches the compiler may contract a
different set of multiplies and adds into FFMA, and an FFMA rounds once where FMUL + FADD round twice.  The
warp emulator cannot see that (it runs the source on the CPU); the SASS can.  This compiles three units
with the library's nvcc flags and reads `nvdisasm -g`:
  * the generic star<3,6> kernel (variant 1),
  * the `--shape` kernel with every structure define the library build uses,
  * the same kernel with the contact, edge, feet and frame counts left at run time (the defines of
    `--runtime` dropped).
For every source line of dial_device.cuh inside the env-step loop (the static-row copy of rollout_warp, as
scripts/sass_sections.py finds it) it counts the FFMA, FMUL and FADD instructions attributed to that line
(the innermost dial_device.cuh line of the inlining chain), per build.  Unrolling changes how many copies
of a line there are, not what each copy is, so a line is flagged when its counts in two builds are not
proportional: its fused/unfused mix differs.  Lines written with __fmaf_rn / __fmul_rn / __fadd_rn are
marked `pinned`.  The last line of the output counts the pinned lines whose mix differs between the
generic and the specialised kernel."""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import sass_sections as ss  # noqa: E402

g = ss.g
KINDS = ("FFMA", "FMUL", "FADD")
PIN = re.compile(r"__f(ma|mul|add)f?_rn\b")


def compile_cubin(flags, out):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + g.NVCC_FLAGS + flags + ["-cubin", "-o", out, os.path.join(g.CSRC, ss.VAR)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(r.stderr)


def line_counts(cubin, hdr, span, func_of):
    """{header line: Counter(opcode with modifiers)} of the fp32 FFMA / FMUL / FADD instructions of the
    env-step loop of the static-row copy of rollout_warp."""
    dis = subprocess.run([os.environ.get("NVDISASM", "/usr/local/cuda/bin/nvdisasm"), "-gi", "-c", cubin],
                         capture_output=True, text=True, check=True).stdout
    insts = ss.parse_sass(dis)
    t0, t1 = span
    last_exit = max(a for a, t, _ in insts if t == "EXIT")
    copies = sorted({ch[-1][1] for a, _, ch in insts if a <= last_exit and ch and ch[-1][0] == ss.VAR
                     and any(f == ss.HDR and func_of.get(n) == "rollout_warp" for f, n in ch)})
    static_row = copies[-1]
    out = collections.defaultdict(collections.Counter)
    for a, text, ch in insts:
        if a > last_exit or not ch or ch[-1] != (ss.VAR, static_row):
            continue
        rw = next((n for f, n in ch if f == ss.HDR and func_of.get(n) == "rollout_warp"), None)
        if rw is None or not (t0 <= rw <= t1):
            continue
        op = re.sub(r"^@!?U?P\w+\s+", "", text).split()[0]
        if op.split(".")[0] not in KINDS:
            continue
        site = tuple(n for f, n in ch if f == ss.HDR)
        if site:
            out[site][op] += 1
    return out


def same_mix(a, b):
    """Counters a and b (both non-empty) are proportional: each copy of the line compiled alike."""
    keys = set(a) | set(b)
    ta, tb = sum(a.values()), sum(b.values())
    return all(a[k] * tb == b[k] * ta for k in keys)


def fmt(c):
    return " ".join(f"{k}:{c[k]}" for k in sorted(c)) or "-"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="go2")
    ap.add_argument("--runtime", default="NCON,NEDGE,NFEET,N_FRAMES",
                    help="DIAL_SHAPE_* fields left at run time in the third build")
    ap.add_argument("--all", action="store_true", help="print every line with fp32 arithmetic, not only the flagged ones")
    args = ap.parse_args()
    defs = dict(g._shape_defines())
    if args.shape not in defs:
        raise SystemExit(f"unknown shape {args.shape!r} (known: {', '.join(defs)})")
    drop = {f"DIAL_SHAPE_{f}" for f in args.runtime.split(",") if f}
    shape_flags = ["-DDIAL_VARIANT=1", f"-DDIAL_SHAPE_NAME={args.shape}"]
    builds = (("generic", ["-DDIAL_VARIANT=1"]),
              (args.shape, shape_flags + [f"-D{d}" for d in defs[args.shape]]),
              (f"{args.shape}-rt", shape_flags + [f"-D{d}" for d in defs[args.shape] if d.split("=")[0] not in drop]))
    hdr = open(os.path.join(g.CSRC, ss.HDR)).read().splitlines()
    func_of = ss.functions_of(hdr)
    span = ss.block_span(hdr, ss.find_line(hdr, func_of, "rollout_warp", r"for \(int t = 0; t < H; \+\+t\) \{"))
    counts = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, flags in builds:
            cubin = os.path.join(tmp, f"{name}.cubin")
            compile_cubin(flags, cubin)
            counts[name] = line_counts(cubin, hdr, span, func_of)
    names = [n for n, _ in builds]
    gen = counts["generic"]
    print(f"fp32 FFMA / FMUL / FADD per {ss.HDR} line of the env-step loop ({ss.HDR}:{span[0]}-{span[1]})")
    print(f"builds: {', '.join(names)} ({names[2]}: {', '.join(sorted(drop))} at run time)\n")
    print("| line | inlined via | source | " + " | ".join(names) + " | note |")
    print("|---|---|---|" + "---|" * len(names) + "---|")
    pinned_diff, flagged = set(), set()
    for site in sorted(set().union(*counts.values())):
        row = [counts[n].get(site, collections.Counter()) for n in names]
        line = site[0]
        pinned = bool(PIN.search(hdr[line - 1]))
        notes = []
        for n, c in zip(names[1:], row[1:]):
            if not c or not row[0]:
                if c or row[0]:
                    notes.append(f"only in {'generic' if row[0] else n}")
            elif not same_mix(row[0], c):
                notes.append(f"mix differs: {n}")
        if pinned:
            notes.append("pinned")
        differs = any(n.startswith("mix differs") for n in notes)
        if differs:
            flagged.add(line)
        if pinned and row[0] and row[1] and not same_mix(row[0], row[1]):
            pinned_diff.add(line)
        if args.all or differs:
            via = " < ".join(str(n) for n in site[1:4]) + (" < ..." if len(site) > 4 else "")
            src = hdr[line - 1].strip()
            print(f"| {line} | {via} | `{src[:60]}` | " + " | ".join(fmt(c) for c in row) + f" | {'; '.join(notes)} |")
    print(f"\nlines whose fused/unfused mix differs from the generic kernel at some site: {len(flagged)} "
          f"{sorted(flagged)}")
    print(f"pinned lines whose mix differs between generic and {args.shape}: {len(pinned_diff)} {sorted(pinned_diff)}")


if __name__ == "__main__":
    main()
