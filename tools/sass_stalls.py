"""Static issue schedule of a kernel's hot loop (development tool): sums the stall counts ptxas encoded in the SASS control words between
two addresses -- the cycles ONE warp needs per pass when nothing but its own fixed-latency dependencies holds it back.
   python tools/sass_stalls.py <lib.so> <mangled-name substring> <lo hex> <hi hex>"""
import collections
import re
import subprocess
import sys


def dump(lib, cuobjdump="cuobjdump"):
    """The SASS listing of every function of `lib`, as lines."""
    return subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True, check=True).stdout.splitlines()


def parse(sass, name):
    """[(address, instruction text, high control word)] of the first function of a dump() listing whose mangled name contains `name`."""
    ins, on, i = [], False, 0
    while i < len(sass):
        l = sass[i]
        if "Function :" in l:
            if on:
                break
            on = name in l
        m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);\s+/\* (0x[0-9a-f]{16}) \*/", l) if on else None
        if m and i + 1 < len(sass):
            m2 = re.match(r"\s+/\* (0x[0-9a-f]{16}) \*/", sass[i + 1])
            if m2:
                ins.append((int(m.group(1), 16), m.group(2).strip(), int(m2.group(1), 16)))
                i += 2
                continue
        i += 1
    return ins


def opcode(text):
    """Opcode with its modifiers ("LDG.E.128.CONSTANT"), the guard predicate stripped."""
    return re.sub(r"^@!?U?P\d+\s+", "", text).split()[0]


def main():
    lib, name, lo, hi = sys.argv[1], sys.argv[2], int(sys.argv[3], 16), int(sys.argv[4], 16)
    ins = parse(dump(lib), name)
    body = [x for x in ins if lo <= x[0] <= hi]
    stalls = [(h >> 41) & 0xF for _, _, h in body]          # control bits 105..108 of the 128-bit instruction
    mix = collections.Counter(opcode(t) for _, t, _ in body)
    print("%s [%#x, %#x]: %d instructions, sum of stall counts %d (%.2f cycles per instruction for a lone warp)" % (name, lo, hi, len(body), sum(stalls), sum(stalls) / max(1, len(body))))
    print("stall-count histogram:", sorted(collections.Counter(stalls).items()))
    print("instruction mix:", ", ".join("%s %d" % kv for kv in mix.most_common(12)))


if __name__ == "__main__":
    main()
