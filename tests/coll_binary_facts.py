"""What the compiler made of libb200coll, read once per test session: the kernel symbols (nm), each kernel's SASS (cuobjdump) and
ptxas's resource report for one source file, compiled with the library's flags."""
import functools
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


@functools.lru_cache(maxsize=None)
def _symbols(lib):
    return subprocess.run(["nm", "-C", lib], capture_output=True, text=True, check=True).stdout


def kernels(lib, key):
    """The demangled names of the symbols of `lib` that contain `key`, sorted, each once."""
    return sorted({l.split(" ", 2)[-1] for l in _symbols(lib).splitlines() if key in l})


def template_args(name):
    """The template arguments of a demangled kernel name, stripped: 'ns::k<a, b>(...)' -> ('a', 'b')."""
    return tuple(a.strip() for a in name.split("<", 1)[1].split(">", 1)[0].split(","))


@functools.lru_cache(maxsize=None)
def sass(lib):
    """{mangled kernel name: its SASS listing} of `lib`."""
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur:
            funcs[cur].append(line)
    return {k: "\n".join(v) for k, v in funcs.items()}


@functools.lru_cache(maxsize=None)
def ptxas(src):
    """ptxas's account of coll/src/<src> compiled with the library's flags: ({mangled kernel: (stack, spill stores, spill loads)},
    {mangled kernel: registers})."""
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([os.environ.get("NVCC", "nvcc"), *NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(ROOT, "coll", "src", src),
                            "-o", os.path.join(d, src + ".o")], capture_output=True, text=True, check=True)
    report, regs, cur = {}, {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            report[cur] = tuple(map(int, m.groups()))
            continue
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            regs[cur] = int(m.group(1))
    return report, regs
