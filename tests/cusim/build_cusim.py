"""Builds tests/cusim/_build/libcloudini_b200_cusim.so — TEST INFRASTRUCTURE ONLY (see cuda_runtime.h here).

The product's kernel sources (cloudini_b200/csrc/*.cu, unmodified on disk) are copied into _build/csrc with three
mechanical rewrites that g++ needs, then compiled against the cusim shim of <cuda_runtime.h>:
  * `kernel<<<grid, block, smem, stream>>>(args);`        -> `cusim::launch(dim3(grid), dim3(block), smem, [&]{ kernel(args); });`
  * `extern __shared__ __align__(16) uint8_t name[];`      -> `uint8_t* const name = (uint8_t*)cusim::dyn_smem();`
  * the five inline-PTX accessors (relaxed / acquire / release global loads and stores, %globaltimer) -> __atomic builtins
The library reports "cusim" in cldn_b200_version(); bench.py and smoke() refuse such a library.
"""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "cloudini_b200", "csrc")
OUT_DIR = os.path.join(HERE, "_build")
GEN = os.path.join(OUT_DIR, "csrc")
LIB = os.path.join(OUT_DIR, "libcloudini_b200_cusim.so")
sys.path.insert(0, ROOT)
from cloudini_b200.build import SOURCES  # noqa: E402  (the same translation units as the product build)

PTX = {
    "ld.relaxed.gpu.global.u64": lambda outs, ins: f"{outs[0]} = __atomic_load_n({ins[0]}, __ATOMIC_RELAXED); ::cusim::poll_yield();",
    "st.relaxed.gpu.global.u64": lambda outs, ins: f"__atomic_store_n({ins[0]}, {ins[1]}, __ATOMIC_RELAXED);",
    "ld.acquire.gpu.global.u32": lambda outs, ins: f"{outs[0]} = __atomic_load_n({ins[0]}, __ATOMIC_ACQUIRE); ::cusim::poll_yield();",
    "st.release.gpu.global.u32": lambda outs, ins: f"__atomic_store_n({ins[0]}, {ins[1]}, __ATOMIC_RELEASE);",
    "ld.acquire.gpu.global.u64": lambda outs, ins: f"{outs[0]} = __atomic_load_n({ins[0]}, __ATOMIC_ACQUIRE); ::cusim::poll_yield();",
    "st.release.gpu.global.u64": lambda outs, ins: f"__atomic_store_n({ins[0]}, {ins[1]}, __ATOMIC_RELEASE);",
    "mov.u64 %0, %globaltimer": lambda outs, ins: f"{outs[0]} = ::cusim::globaltimer_ns();",
    # bfind.u32: position of the most significant set bit, 0xffffffff for 0
    "bfind.u32": lambda outs, ins: f"{outs[0]} = (({ins[0]}) == 0u) ? 0xffffffffu : (31u - static_cast<unsigned>(__builtin_clz({ins[0]})));",
    # shr.b32: shift amounts above 31 are clamped to 32 (result 0), unlike C++
    # lop3.b32 d, a, b, c, immLut: bit i of d = immLut[(a_i << 2) | (b_i << 1) | c_i]; the LUT is part of the template text
    "lop3.b32": lambda outs, ins, tmpl="": f"{outs[0]} = ::cusim::lop3({ins[0]}, {ins[1]}, {ins[2]}, {tmpl.rstrip(';').split(',')[-1].strip()});",
    # bmsk.clamp.b32 d, a, b: b bits set starting at bit a (both clamped to 32)
    "bmsk.clamp.b32": lambda outs, ins: f"{outs[0]} = ::cusim::bmsk_clamp({ins[0]}, {ins[1]});",
    "prefetch.global.L2": lambda outs, ins: "((void)0);",
    "prefetch.global.L1": lambda outs, ins: "((void)0);",
    # cp.async: the kernels compile these only without CLDN_CUSIM (the emulation copies synchronously); still rewritten
    "cp.async.cg.shared.global": lambda outs, ins: "((void)0);",
    "cp.async.ca.shared.global": lambda outs, ins: "((void)0);",
    "cp.async.commit_group": lambda outs, ins: "((void)0);",
    # ld.shared.u32 with a 32-bit shared-window address: device builds only (the sources take the pointer path under CLDN_CUSIM);
    # restated as a trap so that a use that slips through is loud
    "ld.shared.u32": lambda outs, ins: f"{outs[0]} = 0; abort();",
    "cp.async.wait_group": lambda outs, ins: "((void)0);",
    "shl.b32": lambda outs, ins: f"{outs[0]} = (({ins[1]}) > 31u) ? 0u : (static_cast<unsigned>({ins[0]}) << ({ins[1]}));",
    # max.NaN.f32: NaN if either operand is NaN
    "max.NaN.f32": lambda outs, ins: f"{outs[0]} = (std::isnan({ins[0]}) || std::isnan({ins[1]})) ? std::numeric_limits<float>::quiet_NaN() : fmaxf({ins[0]}, {ins[1]});",
    "shr.b32": lambda outs, ins: f"{outs[0]} = (({ins[1]}) > 31u) ? 0u : (static_cast<unsigned>({ins[0]}) >> ({ins[1]}));",
}


def _split_top(s, sep=","):
    parts, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == sep and depth == 0:
            parts.append(cur.strip())
            cur = ""
        else:
            cur += ch
    parts.append(cur.strip())
    return parts


def _rewrite_launches(text, fname):
    out, pos = "", 0
    while True:
        i = text.find("<<<", pos)
        if i < 0:
            return out + text[pos:]
        m = re.search(r"([A-Za-z_][A-Za-z0-9_]*)\s*$", text[pos:i])
        if not m:
            raise RuntimeError(f"{fname}: launch without a plain kernel name near offset {i}")
        name_start = pos + m.start(1)
        j = text.index(">>>", i)
        cfg = _split_top(text[i + 3:j])
        if len(cfg) < 2:
            raise RuntimeError(f"{fname}: launch configuration {cfg}")
        k = j + 3
        while text[k] in " \t":
            k += 1
        if text[k] != "(":
            raise RuntimeError(f"{fname}: launch arguments not found")
        depth, e = 0, k
        while True:
            if text[e] == "(":
                depth += 1
            elif text[e] == ")":
                depth -= 1
                if depth == 0:
                    break
            e += 1
        args = text[k + 1:e]
        smem = cfg[2] if len(cfg) > 2 else "0"
        out += text[pos:name_start]
        out += (f"::cusim::launch(dim3({cfg[0]}), dim3({cfg[1]}), static_cast<size_t>({smem}), [&]() {{ {m.group(1)}({args}); }}, "
                f"reinterpret_cast<const void*>(+{m.group(1)}))")
        pos = e + 1


def _rewrite_asm(text, fname):
    out, pos = "", 0
    while True:
        m = re.compile(r"\basm\s*(?:volatile\s*)?\(").search(text, pos)
        if not m:
            return out + text[pos:]
        k, depth, in_str = m.end() - 1, 0, False
        while True:  # matching parenthesis, string literals skipped
            ch = text[k]
            if in_str:
                if ch == "\\":
                    k += 1
                elif ch == '"':
                    in_str = False
            elif ch == '"':
                in_str = True
            elif ch == "(":
                depth += 1
            elif ch == ")":
                depth -= 1
                if depth == 0:
                    break
            k += 1
        body = text[m.end():k]
        end = k + 1
        while text[end] in " \t":
            end += 1
        assert text[end] == ";", (fname, body)
        tmpl = re.match(r'\s*"([^"]*)"', body)
        if tmpl.group(1).strip() == "":  # compiler barrier: keep it
            out += text[pos:m.start()] + '__asm__ __volatile__("" ::: "memory");'
            pos = end + 1
            continue
        key = next((p for p in PTX if tmpl.group(1).startswith(p)), None)
        if key is None:
            raise RuntimeError(f"{fname}: no cusim restatement for inline PTX `{tmpl.group(1)}`")
        sections = _split_top(body[tmpl.end():], ":")

        def operands(sec):
            return [o[o.index("(") + 1:o.rindex(")")] for o in _split_top(sec) if "(" in o]
        outs = operands(sections[1]) if len(sections) > 1 else []
        ins = operands(sections[2]) if len(sections) > 2 else []
        out += text[pos:m.start()] + (PTX[key](outs, ins, tmpl.group(1)) if key == "lop3.b32" else PTX[key](outs, ins))
        pos = end + 1


def _register_static_shared(text):
    """`__shared__ T a, b[4];` -> the same line + `::cusim::register_shared(&a, sizeof(a)); ...` (see cuda_runtime.h)."""
    out = []
    for line in text.split("\n"):
        m = re.match(r"^(\s*)__shared__\s+(.*);\s*(//.*)?$", line)
        if not m or "extern" in line:
            out.append(line)
            continue
        parts = _split_top(m.group(2))
        names = []
        first = re.match(r"^(.*?)(\w+)\s*((?:\[[^\]]*\])*)$", parts[0].strip())
        names.append(first.group(2))
        for extra in parts[1:]:
            names.append(re.match(r"^\s*(\w+)", extra).group(1))
        out.append(line + " " + " ".join(f"::cusim::register_shared(&{n}, sizeof({n}));" for n in names))
    return "\n".join(out)


def transform(text, fname):
    text = re.sub(r'#include "\.\./\.\./include/(\w+\.h)"', lambda m: f'#include "{os.path.join(ROOT, "include", m.group(1))}"', text)
    text = re.sub(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?uint8_t\s+(\w+)\[\];",
                  r"uint8_t* const \1 = static_cast<uint8_t*>(::cusim::dyn_smem());", text)
    text = re.sub(r"\b__noinline__\b", "__attribute__((noinline))", text)  # a macro of that name would break libstdc++
    text = _rewrite_asm(text, fname)
    text = _rewrite_launches(text, fname)
    text = _register_static_shared(text)
    text = text.replace('"cloudini_b200 0.1.0 (wire v5, sm_90a)"', '"cloudini_b200 0.1.0 cusim (CPU emulation of the CUDA model: TEST ONLY)"')
    return text


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, f) for f in ("cuda_runtime.h", "cusim.cpp", "build_cusim.py")]
    deps += [os.path.join(ROOT, "include", f) for f in ("cloudini_b200.h", "cloudini_b200_ros.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, opt="-O1", asan=False):
    """asan=True builds libcloudini_b200_cusim_asan.so (AddressSanitizer: out-of-bounds accesses of the kernels on
    "device" = heap memory are reported). Load it with LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0."""
    lib = LIB.replace(".so", "_asan.so") if asan else LIB
    if not force and not asan and not needs_build():
        return LIB
    os.makedirs(GEN, exist_ok=True)
    for f in os.listdir(CSRC):
        with open(os.path.join(CSRC, f)) as fh:
            text = fh.read()
        with open(os.path.join(GEN, f), "w") as fh:
            fh.write(transform(text, f))
    flags = ["-std=c++17", opt, "-g", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-pthread", "-I", HERE, "-w"]
    if asan:
        # + alignment: x86 tolerates a misaligned uint4 / uint64 access, the GPU raises "misaligned address"
        # + shift-exponent / float-cast-overflow / integer-divide-by-zero: where C++ leaves the result open the two
        #   machines differ (a shift by >= the width wraps on x86 and clamps on the GPU, an out-of-range float -> int
        #   cast gives INT_MIN on x86 and saturates on the GPU), so emulated parity would prove nothing there
        ub = "alignment,shift-exponent,float-cast-overflow,integer-divide-by-zero"
        flags += ["-fsanitize=address", "-fsanitize=" + ub, "-fno-sanitize-recover=" + ub, "-fno-omit-frame-pointer"]
    procs = []
    for src in SOURCES + ["cusim.cpp"]:
        path = os.path.join(HERE, src) if src == "cusim.cpp" else os.path.join(GEN, src)
        obj = os.path.join(OUT_DIR, os.path.splitext(src)[0] + ("_asan.o" if asan else ".o"))
        cmd = ["g++", *flags, "-x", "c++", "-c", path, "-o", obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out[-6000:])
            raise RuntimeError(f"cusim: g++ failed on {src}")
        objs.append(obj)
    subprocess.check_call(["g++", "-shared", "-pthread", *(["-fsanitize=address", "-fsanitize=alignment,shift-exponent,float-cast-overflow,integer-divide-by-zero"] if asan else []), "-o", lib, *objs, "-ldl"])
    return lib


def build_racecheck():
    """ThreadSanitizer build: tests/cusim/_build/racecheck (an executable: TSAN wants to own the process from the start).
    Kernel sources + C ABI + racecheck_main.cpp are instrumented; the scheduler (cusim.cpp) is not (see the comment there)."""
    os.makedirs(GEN, exist_ok=True)
    for f in os.listdir(CSRC):
        with open(os.path.join(CSRC, f)) as fh:
            text = fh.read()
        with open(os.path.join(GEN, f), "w") as fh:
            fh.write(transform(text, f))
    # -O0: with optimisation gcc's tsan pass drops enough of the kernels' plain loads / stores that the detector's own
    # positive control (racecheck --control-racy) goes silent
    common = ["-std=c++17", "-O0", "-g", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-pthread", "-I", HERE, "-w"]
    procs, objs = [], []
    for src in SOURCES + ["cusim.cpp", "racecheck_main.cpp"]:
        own = src in ("cusim.cpp", "racecheck_main.cpp")
        path = os.path.join(HERE, src) if own else os.path.join(GEN, src)
        obj = os.path.join(OUT_DIR, os.path.splitext(src)[0] + "_tsan.o")
        flags = list(common) + (["-DCUSIM_TSAN=1"] if src == "cusim.cpp" else ["-fsanitize=thread"])
        if src == "racecheck_main.cpp":
            flags += ["-I", os.path.join(ROOT, "include")]
        procs.append((src, obj, subprocess.Popen(["g++", *flags, "-x", "c++", "-c", path, "-o", obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out[-6000:])
            raise RuntimeError(f"cusim: g++ failed on {src}")
        objs.append(obj)
    exe = os.path.join(OUT_DIR, "racecheck")
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, *objs, "-ldl"])
    return exe


if __name__ == "__main__":
    if "--tsan" in sys.argv:
        print(build_racecheck())
    else:
        print(build(force="--force" in sys.argv, asan="--asan" in sys.argv))
