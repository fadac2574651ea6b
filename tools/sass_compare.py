"""Compare the SASS of every kernel in one object file against another, instruction by instruction (no GPU needed).

    python tools/sass_compare.py OLD.o NEW.o

For example, to check that a change leaves the planar local_laplacian kernels alone: build the parent commit's
halide_b200/csrc/local_laplacian.o in a scratch checkout, build this tree's, and compare the two.

Kernels are matched by demangled name.  A template parameter that a change appends with a default value changes the
mangled name of every existing instantiation without changing its code, so the new object's names are also tried with
such trailing defaults removed, one after another: the interleaved-layout parameters `bool IL = false` (ll_level1_kernel;
nl_means_kernel and nl_means_window_kernel, with the frame-walk parameter `bool FR = false` after it),
`int PI = 1, int PO = 1` (ll_up2_kernel), the level set type `typename LS = LevelSet` and after it the stride set type
`typename FS = FrameStrides` (ll_coarse_fused_kernel), and ll_tone_kernel's `typename T = uint16_t, int PI = 1, int PO = 1,
bool FRAMES = false` (its element type, `unsigned short`, is trailing once the others are stripped).  A kernel that gained the frame element type as its
first template parameter is also tried without it when that type is float: `f<float>(` as the plain function `f(` (the
demangled name of a template instance also carries its return type, `void `), `f<float, 3, 7>(` as `f<3, 7>(`
(bg_hist_blurz_kernel, bg_slice_kernel, nl_means_kernel, nl_means_window_kernel; the bilateral_grid kernels also gained
the frame-walk parameter `bool FR = false` after it).  A plain kernel that became a template of one defaulted `bool`
is tried without it: `f<false>(` as `f(` (bg_blur_xy_kernel, bg_hist_blurz_s_kernel, bg_slice_s_kernel, blur3x3_u16_kernel;
blur3x3_u16_quad_kernel<6> and stencil_chain_window_kernel<F> gained `bool FR = false` as a trailing default).  An old kernel
with no new one of its name is also matched by name and template arguments alone, with the parameter list and a last
template argument `0` dropped on both sides (a plain function: by name alone): the template arguments fix the parameter
types however they are spelled (nl_means's and bilateral_grid's kernels take theirs through an alias, which demangles as
`std::conditional<...>::type`), and a std::enable_if choice between overloads adds that `0` (nl_means_window_kernel
before it was one template).  An old frame-walking instance, `f<..., true>(` or `f<true>(`, is also matched by name and
template arguments alone against the kernel without its `bool FR` parameter (blur3x3_u16_kernel and
blur3x3_u16_quad_kernel<6>, which serve one frame and clips alike).  Instruction addresses and padding are
dropped before comparing; opcodes, operands and encodings must match.  Prints each old kernel that is missing or differs, then a count; exits 1 if any.
"""
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
# trailing template arguments that stand for the defaults of appended parameters
DEFAULT_TAILS = [", 1, 1>(", ", false>(", ", llk::LevelSet>(", ", llk::FrameStrides>(", ", unsigned short>("]
# a leading element type parameter: its float instance against the kernel before it had the parameter; and a plain
# kernel's one appended `bool = false`
HEADS = [(re.compile(r"^void (.*)<float>\("), r"\1("), (re.compile(r"<float, "), "<"), (re.compile(r"^void (.*)<false>\("), r"\1(")]
# a name without its parameter list and an enable_if selector argument; a plain function's name without its parameter
# list (the first parenthesis that follows a name character: "(anonymous namespace)" precedes none)
BARE = re.compile(r"(, 0)?>\(.*\)$")
PLAIN = re.compile(r"(?<=\w)\(.*\)$")
# an old frame-walking instance's last template argument, `bool FR = true` (a plain function without it also loses its
# return type, as in HEADS)
FR_TAILS = [(re.compile(r", true>\("), ">("), (re.compile(r"^void (.*)<true>\("), r"\1(")]


def bare(name):
    return BARE.sub(">", name) if BARE.search(name) else PLAIN.sub("", name)


def kernels(obj):
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    res, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                res[name] = body
            name, body = m.group(1), []
        elif name and "/*" in line:
            # (runs of blanks collapsed: cuobjdump pads every line to the longest instruction in the file)
            body.append(" ".join(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).split()))
    if name:
        res[name] = body
    names = list(res)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return {d: res[m] for m, d in zip(names, demangled)}


def main():
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    by_name = {}
    for k, v in new.items():
        by_name.setdefault(k, []).append(v)
        stripped = k
        while any(tail in stripped for tail in DEFAULT_TAILS):  # (several appended defaults: strip them one by one)
            for tail in DEFAULT_TAILS:
                stripped = stripped.replace(tail, ">(")
            by_name.setdefault(stripped, []).append(v)
        for pat, repl in HEADS:
            if pat.search(k):
                by_name.setdefault(pat.sub(repl, k, count=1), []).append(v)
    by_bare = {}
    for k, vs in by_name.items():
        by_bare.setdefault(bare(k), []).extend(vs)
    bad = 0
    for k, v in old.items():
        without_fr = k
        for pat, repl in FR_TAILS:
            without_fr = pat.sub(repl, without_fr, count=1)
        cands = by_name.get(k) or by_bare.get(bare(k)) or by_bare.get(bare(without_fr), [])
        if not any(c == v for c in cands):
            print(("DIFFERS " if cands else "MISSING ") + k)
            bad += 1
    print(f"{len(old) - bad} of {len(old)} kernels of {sys.argv[1]} have identical SASS in {sys.argv[2]} ({len(new)} kernels there)")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
