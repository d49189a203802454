"""Check that every tap step of the tensor-core convolution compiles to one wgmma commit group.

    python tools/check_wgmma_groups.py [--lib vtoonify_b200/lib/libvtoonify_b200.so] [--log build.log] [--kernel conv_wgrad_kernel]

conv_tc_kernel keeps one wgmma group in flight while it waits for the next pipeline stage. That only works when ptxas keeps
each step's MMAs in one hardware group. When it cannot (runtime control flow between wgmma.fence and wgmma.commit_group, or
a printf anywhere in the kernel), it splits the step and closes it with a placeholder HGMMA. The wait for "all but one
group" then waits for the step's own MMAs, and the tensor pipe drains at every step. Results are still correct; only the
speed drops. The symptoms in the SASS (cuobjdump -sass of the built library), for every instantiation of the kernel (--kernel,
default conv_tc_kernel; the weight-gradient kernel conv_wgrad_kernel follows the same one-group-per-step rule):

  * a placeholder HGMMA, which writes RZ (`HGMMA.64x8x16.F16 RZ, gdesc[URZ], RZ, !UPT, gsb0`);
  * an HGMMA that closes a group (`gsb0`) and is followed by another HGMMA before any `WARPGROUP.DEPBAR` (wait).

With --log, a build log of `VT_PTXAS_V=1 vtoonify_b200/csrc/build.sh` is also checked for ptxas' C7519 notice
("warpgroup.arrive is injected ...") on that kernel.

An instantiation that moves registers between its warpgroups (setmaxnreg: `USETMAXREG.DEALLOC` in warpgroup 0, the producer
and transform warps, and `USETMAXREG.TRY_ALLOC` in the two consumer warpgroups) is also checked against the register count
the launch allocates (`cuobjdump -res-usage`): 128 * dec + 256 * inc must not exceed 384 * REG, and the instantiation must not
spill. `setmaxnreg.inc` waits until enough registers are free, so a plan above the allocation hangs instead of failing.
Exit status 0 when every check passes, 1 otherwise.
"""
import argparse
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "vtoonify_b200", "lib", "libvtoonify_b200.so")
KERNEL = "conv_tc_kernel"

_INSN = re.compile(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([^;]*);")


def find_cuobjdump():
    """cuobjdump from PATH, else from the CUDA toolkit ($CUDA_HOME, /usr/local/cuda); None when there is none."""
    found = shutil.which("cuobjdump")
    if found:
        return found
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.access(os.path.join(home, "bin", "cuobjdump"), os.X_OK):
            return os.path.join(home, "bin", "cuobjdump")
    return None


def short_name(mangled, kernel=KERNEL):
    m = re.search(kernel + r"I((?:Li\d+E)+)E", mangled)
    if not m:
        return mangled
    return kernel + "<" + ", ".join(re.findall(r"Li(\d+)E", m.group(1))) + ">"


def kernel_sass(sass_text, kernel=KERNEL):
    """{function name: [instruction text]} for every instantiation of `kernel` in a cuobjdump -sass listing."""
    funcs, cur = {}, None
    for line in sass_text.splitlines():
        if "Function :" in line:
            name = line.split("Function :", 1)[1].strip()
            cur = funcs.setdefault(name, []) if kernel in name else None
        elif cur is not None:
            m = _INSN.search(line)
            if m:
                cur.append(m.group(1).strip())
    return funcs


def check_groups(insns):
    """(number of HGMMAs, number of groups, [problems]) of one function's instruction stream."""
    problems, n_mma, n_groups, open_gsb0 = [], 0, 0, False
    for i, ins in enumerate(insns):
        if ins.startswith("WARPGROUP.DEPBAR"):
            open_gsb0 = False
        elif ins.startswith("HGMMA"):
            if re.match(r"HGMMA\.\S+\s+RZ\b", ins):
                problems.append(f"placeholder group at instruction {i}: {ins}")
            if open_gsb0:
                problems.append(f"group closed by gsb0 and followed by another HGMMA without a wait at instruction {i}: {ins}")
            n_mma += 1
            open_gsb0 = "gsb0" in ins
            n_groups += open_gsb0
    return n_mma, n_groups, problems


_MAXREG = re.compile(r"USETMAXREG\.(DEALLOC|TRY_ALLOC)\.CTAPOOL\s+(?:U?P\w+\s*,\s*)?(0x[0-9a-f]+|\d+)")
_RES = re.compile(r"Function\s+(\S+?):\s*REG:(\d+)\s+STACK:(\d+)\s+SHARED:\d+\s+LOCAL:(\d+)")
THREADS, XFORM_THREADS, CONSUMER_THREADS = 384, 128, 256


def maxreg_plan(insns):
    """(dec, inc) register counts of the setmaxnreg instructions of one function; None for either that is absent."""
    dec = inc = None
    for ins in insns:
        m = _MAXREG.search(ins)
        if m:
            v = int(m.group(2), 0)
            if m.group(1) == "DEALLOC":
                dec = v
            else:
                inc = v
    return dec, inc


def res_usage(text):
    """{function name: (REG, STACK, LOCAL)} from a cuobjdump -res-usage listing."""
    return {m.group(1): (int(m.group(2)), int(m.group(3)), int(m.group(4))) for m in _RES.finditer(text)}


def check_regs(insns, usage):
    """[problems] of one function's register reallocation; usage = (REG, STACK, LOCAL) or None. Empty without setmaxnreg."""
    dec, inc = maxreg_plan(insns)
    if dec is None and inc is None:
        return []
    if dec is None or inc is None:
        return [f"setmaxnreg plan incomplete (dec {dec}, inc {inc})"]
    if usage is None:
        return ["no -res-usage entry for the function"]
    reg, stack, local = usage
    problems = []
    if XFORM_THREADS * dec + CONSUMER_THREADS * inc > THREADS * reg:
        problems.append(f"setmaxnreg plan {XFORM_THREADS} x {dec} + {CONSUMER_THREADS} x {inc} = "
                        f"{XFORM_THREADS * dec + CONSUMER_THREADS * inc} registers exceeds the launch's {THREADS} x {reg} = {THREADS * reg}")
    if stack or local:
        problems.append(f"spills ({stack} bytes stack, {local} bytes local)")
    return problems


def check_log(log_text, kernel=KERNEL):
    return [line.strip() for line in log_text.splitlines() if "C7519" in line and kernel in line]


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", default=DEFAULT_LIB, help="the built shared library")
    ap.add_argument("--log", default=None, help="build log of VT_PTXAS_V=1 vtoonify_b200/csrc/build.sh")
    ap.add_argument("--kernel", default=KERNEL, help="kernel (template) name whose instantiations are checked")
    args = ap.parse_args(argv)

    tool = find_cuobjdump()
    if tool is None:
        print("check_wgmma_groups: cuobjdump not found", file=sys.stderr)
        return 2
    if not os.path.exists(args.lib):
        print(f"check_wgmma_groups: {args.lib} does not exist (build it first)", file=sys.stderr)
        return 2
    sass = subprocess.run([tool, "-sass", args.lib], capture_output=True, text=True, check=True).stdout
    funcs = kernel_sass(sass, args.kernel)
    usage = res_usage(subprocess.run([tool, "-res-usage", args.lib], capture_output=True, text=True, check=True).stdout)
    failed = False
    if not funcs:
        print(f"FAIL: no {args.kernel} in {args.lib}")
        failed = True
    for name in sorted(funcs, key=lambda n: short_name(n, args.kernel)):
        n_mma, n_groups, problems = check_groups(funcs[name])
        if n_mma == 0:
            problems.append("no HGMMA instructions")
        problems += check_regs(funcs[name], usage.get(name))
        dec, inc = maxreg_plan(funcs[name])
        regs = f", setmaxnreg {dec}/{inc} of {usage[name][0]}" if dec is not None and name in usage else ""
        print(f"{'FAIL' if problems else 'ok  '} {short_name(name, args.kernel)}: {n_mma} HGMMA, {n_groups} groups{regs}")
        for p in problems:
            print(f"       {p}")
        failed = failed or bool(problems)
    if args.log:
        with open(args.log) as f:
            notices = check_log(f.read(), args.kernel)
        for line in notices:
            print(f"FAIL ptxas: {line}")
        failed = failed or bool(notices)
    return 1 if failed else 0


if __name__ == "__main__":
    sys.exit(main())
