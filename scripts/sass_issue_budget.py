"""Per-warp issue budget of the config-2 HMC loop (hmc_run_kernel<ISO, NONE, 4, 2, 128, …, PW = 2>) from its SASS.

Usage: python scripts/sass_issue_budget.py <obj.o> [L] [hmcx_hmc.cu the object was built from] [kernel substring]

The object is hmcx_hmc.cu compiled with the library's flags (hamiltorch_b200/build.py) and -lineinfo.  Like
sass_loop_count.py it reads nvdisasm's listing, but it counts one iteration of one warp along the accept path:
  * the compute loop is the backward branch whose body holds the slot-full barrier (BAR.SYNC 0x2); the producer loop
    the one whose body holds the slot-full arrive (BAR.ARV 0x2);
  * the step loop (the backward branch nested in the compute loop) is weighted by its trips at L, (L - 1) // 2, since
    trajectory_groups peels the first step; of the two paths after it, the one with the odd last step is taken when
    L - 1 is odd;
  * cold blocks are left out: the divergent fall-backs of the shuffles (BRA.DIV targets), the reject branch with the
    :1018 restore (the `else` of the MH test), the producers' log-uniform refill (once per 32 iterations), and for
    the compute warps other than warp 0 the lead thread's scalar stores.  A block is cold when it holds a line of a
    cold source range, or when every block that enters it (back edges aside) is cold.
Prints the weighted counts and opcode histograms as one JSON object."""
import collections, json, os, re, subprocess, sys, tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
obj = sys.argv[1]
L = int(sys.argv[2]) if len(sys.argv) > 2 else 10
SRC = sys.argv[3] if len(sys.argv) > 3 else os.path.join(HERE, '..', 'hamiltorch_b200', 'csrc', 'hmcx_hmc.cu')
pat = sys.argv[4] if len(sys.argv) > 4 else 'hmc_run_kernelILi0ELi0ELi4ELi2ELi128ELb0ELb1ELi1ELb0ELi2E'

# ---- cold source ranges of hmcx_hmc.cu, found by brace matching from marker lines ----
src = open(SRC).read().splitlines()


def block_range(i):
    """1-based line range of the brace block opened on (0-based) line i"""
    depth, j = 0, i
    while True:
        depth += src[j].count('{') - src[j].count('}')
        if depth <= 0 and j > i or (depth == 0 and '{' in src[j] and j >= i and src[j].count('}') >= 1 and j > i):
            return (i + 1, j + 1)
        j += 1


kern = next(i for i, l in enumerate(src) if re.match(r'hmc_run_kernel\(const RunArgs a\)', l))
loop = next(i for i in range(kern, len(src)) if 'for (int n = a.it0' in src[i])
rej = next(i for i in range(loop, len(src)) if '++rejected;' in src[i])
rej_open = next(i for i in range(rej, loop, -1) if src[i].rstrip().endswith('{'))
lead = next(i for i in range(loop, len(src)) if re.search(r'\bif \(lead\) \{', src[i]))
prod = next(i for i, l in enumerate(src) if 'void hmc_produce(' in l)
refill = next(i for i in range(prod, len(src)) if 'if (phase == 0)' in src[i])
COLD = {'reject': block_range(rej_open), 'lead': block_range(lead), 'refill': (refill + 1, refill + 1)}

# ---- the kernel's instructions with line info ----
tmp = tempfile.mkdtemp()
subprocess.check_call(['cuobjdump', '-xelf', 'all', os.path.abspath(obj)], cwd=tmp, stdout=subprocess.DEVNULL)
cubin = [f for f in os.listdir(tmp) if f.endswith('.cubin')][0]
txt = subprocess.run(['nvdisasm', '--print-line-info', os.path.join(tmp, cubin)], capture_output=True,
                     text=True).stdout.splitlines()
start = next(i for i, l in enumerate(txt) if l.startswith('.text.') and pat in l)
insts, labels, pend, cur = [], {}, [], None
for l in txt[start + 1:]:
    if l.startswith('\t.section') or l.startswith('.text.'):
        break
    m = re.search(r'//## File "([^"]+)", line (\d+)', l)
    if m:
        cur = (os.path.basename(m.group(1)), int(m.group(2)))
        continue
    m = re.match(r'\s*(\.L_x_\d+):', l)
    if m:
        pend.append(m.group(1))
        continue
    m = re.match(r'\s+/\*([0-9a-f]{4,5})\*/\s+(\S.*?);', l)
    if m:
        a = int(m.group(1), 16)
        for p in pend:
            labels[p] = a
        pend = []
        insts.append((a, m.group(2), cur))
addr = [a for a, _, _ in insts]
idx = {a: i for i, a in enumerate(addr)}


def op(t):
    w = t.split()
    return w[1] if w[0].startswith('@') else w[0]


def target(t):
    m = re.search(r'BRA.*`\((\.L_x_\d+)\)', t)
    return labels.get(m.group(1)) if m else None


# basic blocks: leaders are labels and the instructions after a branch / exit
leaders = {addr[0]} | set(labels.values())
for i, (a, t, _) in enumerate(insts):
    if (op(t).startswith('BRA') or op(t) == 'EXIT') and i + 1 < len(insts):
        leaders.add(addr[i + 1])
lead_list = sorted(x for x in leaders if x in idx)
blocks = {}
for b, s in enumerate(lead_list):
    e = lead_list[b + 1] if b + 1 < len(lead_list) else addr[-1] + 16
    blocks[s] = [i for i in range(idx[s], len(insts)) if addr[i] < e]


def succ(s):
    last = insts[blocks[s][-1]][1]
    out = []
    tg = target(last)
    if tg is not None:
        out.append(tg)
    uncond = (op(last) == 'BRA' and not last.startswith('@')) or (op(last) == 'EXIT' and not last.startswith('@'))
    nxt = addr[blocks[s][-1]] + 16
    if not uncond and nxt in blocks:
        out.append(nxt)
    return out


# loop back edges; the out-of-line shuffle fall-backs after the last EXIT branch back into the loops and are not loops
last_exit = max(a for a, t, _ in insts if op(t) == 'EXIT')
backs = [(target(t), a) for a, t, _ in insts
         if op(t).startswith('BRA') and target(t) is not None and target(t) < a and a < last_exit]


def loop_with(marker):
    c = [(s, e) for s, e in backs if any(marker(insts[i][1]) for i in range(idx[s], idx[e] + 1))]
    return min(c, key=lambda b: b[1] - b[0])


def count(span, cold_names, weight_inner=True):
    s0, e0 = span
    inside = [s for s in blocks if s0 <= s <= e0]
    inner = [b for b in backs if b != span and s0 <= b[0] and b[1] <= e0]
    trips = (L - 1) // 2
    cold = set()
    for s in inside:
        for i in blocks[s]:
            f, ln = insts[i][2] or ('', 0)
            if f == 'hmcx_hmc.cu' and any(COLD[n][0] <= ln <= COLD[n][1] for n in cold_names):
                cold.add(s)
    for s in blocks:                                       # divergent fall-backs of the shuffles
        last = insts[blocks[s][-1]][1]
        if op(last) == 'BRA.DIV':
            cold.add(target(last))
    # the step loop's tail: the two paths from the first branch after the inner loop's exit to their merge
    for ib in inner:
        after = addr[idx[ib[1]] + 1]
        br = next(s for s in sorted(blocks) if s >= after and target(insts[blocks[s][-1]][1]) is not None)
        tk, ft = target(insts[blocks[br][-1]][1]), addr[blocks[br][-1]] + 16

        def path(p):
            out = []
            while p in blocks and p <= e0:
                out.append(p)
                last = insts[blocks[p][-1]][1]
                if op(last) == 'BRA' and not last.startswith('@'):
                    return out, target(last)
                p = addr[blocks[p][-1]] + 16
            return out, p
        pa, ma = path(ft)
        pb, mb = path(tk)
        pa = [p for p in pa if p not in pb and p < mb]
        flops = lambda ps: sum(op(insts[i][1]) in ('FMUL', 'FFMA') for p in ps for i in blocks[p])
        odd, even = (pa, pb) if flops(pa) > flops(pb) else (pb, pa)
        cold.update(even if (L - 1) % 2 else odd)
    preds = collections.defaultdict(set)
    for s in inside:
        for t in succ(s):
            if t is not None and t > s:
                preds[t].add(s)
    changed = True
    while changed:
        changed = False
        for s in sorted(inside):
            if s not in cold and s != s0 and preds[s] and preds[s] <= cold:
                cold.add(s)
                changed = True
    hist, n = collections.Counter(), 0
    for s in inside:
        if s in cold:
            continue
        w = trips if weight_inner and any(b[0] <= s <= b[1] for b in inner) else 1
        for i in blocks[s]:
            hist[op(insts[i][1])] += w
            n += w
    return n, dict(sorted(hist.items(), key=lambda kv: -kv[1]))


comp = loop_with(lambda t: 'BAR.SYNC' in t and ' 0x2,' in t)
prodl = loop_with(lambda t: 'BAR.ARV' in t and ' 0x2,' in t)
w0, h0 = count(comp, ['reject'])
wk, hk = count(comp, ['reject', 'lead'])
pn, ph = count(prodl, ['refill'])
out = {'kernel': pat, 'L': L,
       'compute_warp0': w0, 'compute_other_warps': wk, 'producer_warp': pn,
       'hist_compute_warp0': h0, 'hist_compute_other_warps': hk, 'hist_producer': ph}
out['per_scheduler'] = w0 + wk + pn      # 2 compute warps (warp 0 of one chain) + 1 producer warp per SM scheduler
print(json.dumps(out))
