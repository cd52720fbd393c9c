"""SASS opcode histogram per kernel of libpulse_b200.so (cuobjdump -sass): evidence of WHICH hardware paths each kernel uses
(HGMMA = wgmma.mma_async, UTMALDG / UTMAREDG = TMA tensor load / reduction, UBLKCP = bulk async copy, ...).

    python tools/sass_histogram.py > sass_histogram.txt
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY = ("UTCHMMA", "UTCBAR", "UTCCP", "LDTM", "STTM", "UTMALDG", "UTMASTG", "UTMAREDG", "UTMAPF", "UTMACCTL", "UBLKCP", "UBLKRED", "SYNCS", "REDG", "ATOMG", "RED",
       "ATOM", "HMMA", "SHFL", "LDS", "STS", "LDG", "STG", "MUFU", "BAR", "ELECT", "FENCE", "ERRBAR", "ACQBULK", "CCTL")


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "pulse_b200", "libpulse_b200.so")
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = collections.Counter()
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m and cur is not None:
            kernels[cur][m.group(1)] += 1
    demangle = subprocess.run(["c++filt"], input="\n".join(kernels), capture_output=True, text=True).stdout.splitlines()
    print(f"# {os.path.relpath(lib, ROOT)}: {len(kernels)} kernels; columns: total instructions | selected opcode families (count)")
    for (name, cnt), dm in zip(kernels.items(), demangle):
        short = re.sub(r"\(anonymous namespace\)::|pulse::", "", dm)
        short = re.sub(r"\(.*", "", short)[:90]
        fam = collections.Counter()
        for op, c in cnt.items():
            base = op.split(".")[0]
            for k in KEY:
                if base == k or (k in ("UTCHMMA", "UTMALDG", "UTMAREDG", "UBLKCP", "LDTM") and base.startswith(k)):
                    fam[op if k in ("UTCHMMA", "UTMALDG", "UTMAREDG", "UBLKCP", "LDTM", "UTCBAR") else k] += c
                    break
        fams = "  ".join(f"{k}:{v}" for k, v in sorted(fam.items(), key=lambda kv: (-kv[1], kv[0])))
        print(f"{short:92s} {sum(cnt.values()):6d} | {fams}")


if __name__ == "__main__":
    main()
