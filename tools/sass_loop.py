"""Static look at the steady-state loop of the 2D cluster kernel in a built library (no GPU needed).

    python tools/sass_loop.py <lib.so> [kernel-substring]    (default: the <5,4,8,false,false,forward> instantiation)

Prints: registers / spills are in ptxas.log; here the SASS of the kernel is split at its back edges, the longest loop body
(two propagation steps) is taken, and its instruction mix, the positions of the exchange instructions (SYNCS wait /
arrive, STS, STAS, LDS, SHFL) along the instruction stream and the share of FFMAs that can take an operand from the
reuse cache are listed.
"""
import collections
import re
import subprocess
import sys


def kernel_sass(lib, pattern):
    txt = subprocess.run(['cuobjdump', '-sass', lib], capture_output=True, text=True, check=True).stdout
    out, on = [], False
    for line in txt.splitlines():
        if 'Function :' in line:
            on = pattern in line
            continue
        if on:
            m = re.search(r'/\*([0-9a-f]{4,6})\*/\s+(.*?);', line)
            if m:
                out.append((int(m.group(1), 16), m.group(2).strip()))
    return out


def opcode(s):
    s = re.sub(r'^@!?U?P\d+\s+', '', s)
    return s.split()[0].split('.')[0]


def main():
    lib = sys.argv[1]
    pat = sys.argv[2] if len(sys.argv) > 2 else 'cspn2d_cluster_kernelILi5ELi4ELi8ELb0ELb0ELi0'
    ins = kernel_sass(lib, pat)
    if not ins:
        raise SystemExit('kernel not found')
    addr = {a: i for i, (a, _) in enumerate(ins)}
    # the task loop is the outermost back edge; the step loop is the longest remaining back edge that contains FFMAs
    loops = []
    for i, (a, s) in enumerate(ins):
        m = re.search(r'BRA(?:\.U)?(?:\.ANY)?\s+(?:!?U?P\d+,\s*)?(0x[0-9a-f]+)', s)
        if m:
            t = int(m.group(1), 16)
            if t in addr and addr[t] < i:
                loops.append((addr[t], i))
    loops = [l for l in loops if l[1] - l[0] > 100]
    loops.sort(key=lambda l: l[1] - l[0])
    cand = [l for l in loops if sum('FFMA' in ins[k][1] for k in range(l[0], l[1] + 1)) >= 300]
    lo, hi = cand[0]          # the shortest loop holding >= 300 FFMAs = the two-step body (2 x 160)
    body = ins[lo:hi + 1]
    print(f'{lib}: kernel has {len(ins)} instructions; step loop = [{lo}, {hi}] ({len(body)} instructions, 2 steps)')
    mix = collections.Counter(opcode(s) for _, s in body)
    print('mix:', ', '.join(f'{k} {v}' for k, v in mix.most_common()))
    n_ffma = mix['FFMA']
    reuse_flag = sum(1 for _, s in body if 'FFMA' in s and '.reuse' in s)
    pred = sum(1 for _, s in body if 'FFMA' in s and s.startswith('@'))
    print(f'FFMA {n_ffma}: {reuse_flag} carry a .reuse flag, {pred} predicated; non-FFMA {len(body) - n_ffma}')
    # event positions
    ev = []
    f = 0
    for k, (a, s) in enumerate(body):
        op = opcode(s)
        if op == 'FFMA':
            f += 1
            continue
        if op in ('SYNCS', 'STS', 'STAS', 'LDS', 'SHFL', 'BAR', 'WARPSYNC', 'FSEL', 'BRA', 'NANOSLEEP'):
            ev.append(f'{k}:{op}{"." + s.split()[0].split(".", 1)[1] if "." in s.split()[0] and op in ("SYNCS", "LDS", "STS") else ""}@{f}')
    print('non-FFMA events as index:op@ffmas-issued-so-far')
    line = ''
    for e in ev:
        if len(line) + len(e) > 150:
            print('  ' + line)
            line = ''
        line += e + '  '
    print('  ' + line)


if __name__ == '__main__':
    main()


def rf_cycles(body):
    """Register-file model of /opt/skills/guides/B300_MICROARCH.md ('RF banking'): an instruction needs
    max(1, #distinct even source registers not in the reuse cache, #distinct odd ones) issue cycles; an operand slot's
    reuse cache holds the register the previous instruction of the warp read there with the .reuse flag."""
    cached = [None, None, None]
    total = ffma = ffma_cycles = 0
    hist = collections.Counter()
    for _, s in body:
        s2 = re.sub(r'^@!?U?P\d+\s+', '', s)
        parts = s2.split(None, 1)
        ops = [o.strip() for o in parts[1].split(',')] if len(parts) > 1 else []
        srcs = ops[1:4] if opcode(s) in ('FFMA', 'FMUL', 'FADD') else ops[1:]
        even, odd = set(), set()
        new_cached = [None, None, None]
        for slot, o in enumerate(srcs[:3]):
            m = re.match(r'[-|~]*R(\d+)(\.reuse)?', o)
            if not m:
                continue
            r = int(m.group(1))
            if cached[slot] != r:
                (even if r % 2 == 0 else odd).add(r)
            if m.group(2):
                new_cached[slot] = r
        cached = new_cached
        c = max(1, len(even), len(odd))
        total += c
        if opcode(s) == 'FFMA':
            ffma += 1
            ffma_cycles += c
            hist[c] += 1
    return total, ffma, ffma_cycles, hist
