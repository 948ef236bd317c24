"""Compare two builds of libssb200.so where the ResNet-18 host refactor must leave them equal (runs on the host, no GPU).

    python scratch/rn_build_diff.py lib_a.so lib_b.so

1. Registers, stack, local and shared memory (cuobjdump -res-usage) of every rn_conv_kernel, srn_dw_kernel,
   srn_dx_kernel and maxpool instance.
2. The SASS of every rn_conv_kernel instance, addresses and comments stripped.
3. ssb_smt_resnet18_train_workspace_bytes and ssb_resnet18_train_workspace_bytes over a grid of shapes, each build
   loaded by SSB200_LIB in a process of its own.
Prints one line per difference and exits 1 if there is any.
"""
import ctypes
import itertools
import json
import os
import re
import subprocess
import sys

KERNELS = re.compile(r"rn_conv_kernel|srn_dw_kernel|srn_dx_kernel|maxpool")
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
BS = (0, 1, 7, 1024, 65535)
HWS = ((1, 1), (65, 26), (65, 69), (256, 256))


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    return dict(zip(names, out.splitlines()))


def res_usage(lib):
    """{kernel: 'REG:.. STACK:.. SHARED:.. LOCAL:..'} of the kernels above."""
    text = subprocess.run([CUOBJDUMP, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\n\s*(REG:\d+ STACK:\d+ SHARED:\d+ LOCAL:\d+)", text)
    names = demangle([f for f, _ in found])
    return {names[f]: u for f, u in found if KERNELS.search(names[f])}


def sass(lib):
    """{rn_conv_kernel instance: its instructions}."""
    text = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur and (ins := re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;", line)):
            out[cur].append(ins.group(1))
    names = demangle(list(out))
    return {names[f]: v for f, v in out.items() if "rn_conv_kernel" in names[f] and "srn" not in names[f]}


def workspace_child():
    lib = ctypes.CDLL(os.environ["SSB200_LIB"])
    smt, tv = lib.ssb_smt_resnet18_train_workspace_bytes, lib.ssb_resnet18_train_workspace_bytes
    smt.restype = tv.restype = ctypes.c_int64
    res = {}
    for B, (H, W), L, n_out in itertools.product(BS, HWS, (0, 21), (1, 2)):
        res[f"smt B={B} {H}x{W} L={L} n_out={n_out}"] = smt(B, H, W, L, n_out)
        res[f"tv B={B} {H}x{W} n_out={n_out}"] = tv(B, H, W, n_out)
    print(json.dumps(res))


def workspace(lib):
    env = dict(os.environ, SSB200_LIB=os.path.abspath(lib))
    out = subprocess.run([sys.executable, __file__, "--workspace-child"], env=env, capture_output=True, text=True,
                         check=True).stdout
    return json.loads(out)


def compare(what, a, b):
    diffs = 0
    for k in sorted(set(a) | set(b)):
        if a.get(k) != b.get(k):
            diffs += 1
            print(f"DIFF {what} {k}: {a.get(k) if what != 'sass' else len(a.get(k) or [])} vs "
                  f"{b.get(k) if what != 'sass' else len(b.get(k) or [])}")
    print(f"{what}: {len(set(a) | set(b))} entries, {diffs} differ")
    return diffs


def main():
    if "--workspace-child" in sys.argv:
        return workspace_child()
    lib_a, lib_b = sys.argv[1:3]
    ua, ub = res_usage(lib_a), res_usage(lib_b)
    for k in sorted(ua):
        print(f"{ua[k]}  {k}")
    n = compare("res-usage", ua, ub)
    n += compare("sass", sass(lib_a), sass(lib_b))
    n += compare("workspace-bytes", workspace(lib_a), workspace(lib_b))
    sys.exit(1 if n else 0)


if __name__ == "__main__":
    main()
