"""Per-kernel SASS statistics of the shipped library: instruction count / code bytes and an opcode histogram of the
instructions that prove the memory path (UBLKCP = 1-D TMA bulk copy, LDGSTS = cp.async, SYNCS = mbarrier, DFMA...).

    python tools/sass_stats.py [LIB] [--json]
    python tools/sass_stats.py [LIB] --local SUBSTRING
    python tools/sass_stats.py --diff OLD_LIB NEW_LIB

--local lists the local-memory instructions (STL / LDL: stack frame and register spills) of every kernel whose mangled or
demangled name contains SUBSTRING, counted per source file and line. The library is built with -lineinfo, so nvdisasm
--print-line-info attributes each instruction to the source line it came from (for inlined code, the line of the inlined
function itself). A device function called out of line is placed inside the section of each kernel that calls it; its
instructions are listed apart, under the function's name."""
import re, subprocess, sys, collections, json, os, tempfile


def short(k):
    out = subprocess.run(["c++filt", k], capture_output=True, text=True).stdout.strip()
    out = re.sub(r'lk::\(anonymous namespace\)::', '', out)
    return re.sub(r'\(.*', '', out)[:80]


def local_report(so, pat):
    """{kernel: {part: Counter((op, file, line) -> count)}} for the kernels matching pat; part "" is the kernel's own body,
    any other part a function it calls out of line."""
    res = collections.OrderedDict()
    with tempfile.TemporaryDirectory() as td:
        subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(so)], cwd=td, check=True, capture_output=True)
        for cub in sorted(f for f in os.listdir(td) if f.endswith(".cubin")):
            txt = subprocess.run(["nvdisasm", "--print-line-info", os.path.join(td, cub)], capture_output=True,
                                 text=True).stdout
            fn, part, where = None, "", ("?", 0)
            for l in txt.splitlines():
                m = re.match(r'^\.text\.(\S+):$', l)
                if m:
                    name = m.group(1)
                    fn = name if (pat in name or pat in short(name)) else None
                    if fn: res.setdefault(fn, collections.OrderedDict())
                    part, where = "", ("?", 0)
                    continue
                m = re.match(r'^\$(\S+):$', l)  # a callee's code inside this section: $<kernel>$<callee> or $__internal_..
                if m:
                    part = m.group(1).split("$")[-1]
                    continue
                m = re.match(r'\s*//## File "([^"]+)", line (\d+)', l)
                if m:
                    where = (os.path.basename(m.group(1)), int(m.group(2)))
                    continue
                m = re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?((?:STL|LDL)\b[A-Z0-9_.]*)', l)
                if fn and m:
                    res[fn].setdefault(part, collections.Counter())[(m.group(1).split('.')[0], where[0], where[1])] += 1
    return res


def sass_by_function(so):
    """{mangled name, anonymous-namespace hash normalised: ([opcode of every instruction], [every SASS line])}"""
    txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    anon = lambda m: "%d_GLOBAL__N__%s" % (len("_GLOBAL__N__" + m.group(1)), m.group(1))  # keeps the name demangleable
    txt = re.sub(r'\d+_GLOBAL__N__[0-9a-f]{8}_\d+_(\w+?_cu)_[0-9a-f]{8}', anon, txt)
    res, name = collections.OrderedDict(), None
    for l in txt.splitlines():
        m = re.search(r'Function : (\S+)', l)
        if m:
            name = m.group(1); res[name] = ([], []); continue
        if name is None: continue
        res[name][1].append(l.strip())
        m = re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)', l)
        if m: res[name][0].append(m.group(1))
    return res


def diff(old_so, new_so):
    old, new = sass_by_function(old_so), sass_by_function(new_so)
    same = 0
    for k in list(old) + [k for k in new if k not in old]:
        if k in old and k in new and old[k][1] == new[k][1]:
            same += 1; continue
        n_old, n_new = (len(d[k][0]) if k in d else None for d in (old, new))
        ops = "only in " + ("new" if n_old is None else "old") if None in (n_old, n_new) else \
            "same opcodes" if collections.Counter(old[k][0]) == collections.Counter(new[k][0]) else "opcodes differ"
        print("%-70s %6s -> %-6s %s" % (short(k)[:70], n_old, n_new, ops))
    print("%d of %d functions byte-identical" % (same, len(set(old) | set(new))))


def main():
    args = sys.argv[1:]
    if "--diff" in args:
        i = args.index("--diff")
        return diff(args[i + 1], args[i + 2])
    pat = None
    if "--local" in args:
        i = args.index("--local")
        pat = args[i + 1]
        del args[i:i + 2]
    pos = [a for a in args if not a.startswith("--")]
    so = pos[0] if pos else "leg-kilo_b200/liblegkilo_b200.so"
    if pat is not None:
        rep = local_report(so, pat)
        if not rep:
            sys.exit("no function matches %r" % pat)
        for fn, parts in rep.items():
            print("%s\n  %s" % (short(fn), fn))
            if not parts: print("  no STL / LDL")
            for part, c in parts.items():
                stl = sum(v for (op, _, _), v in c.items() if op == "STL")
                ldl = sum(v for (op, _, _), v in c.items() if op == "LDL")
                print("  %s: %d STL, %d LDL" % ("kernel body" if not part else "called " + short(part), stl, ldl))
                lines = collections.defaultdict(collections.Counter)
                for (op, f, ln), v in c.items(): lines[(f, ln)][op] += v
                for (f, ln) in sorted(lines):
                    print("    %-24s %5d   STL %3d  LDL %3d" % (f, ln, lines[(f, ln)]["STL"], lines[(f, ln)]["LDL"]))
        return
    sass = sass_by_function(so)
    cnt = collections.OrderedDict((k, len(v[0])) for k, v in sass.items())
    ops = {k: collections.Counter(op.split('.')[0] for op in v[0]) for k, v in sass.items()}
    rows = []
    KEYS = ["UBLKCP", "UTMALDG", "LDGSTS", "SYNCS", "DFMA", "DMUL", "DADD", "SHFL", "LDG", "STG", "LDS", "STS", "BAR", "ATOMG", "RED", "MUFU", "CALL"]
    for k, v in sorted(cnt.items(), key=lambda kv: -kv[1]):
        if v < 64: continue
        r = dict(kernel=short(k), instructions=v, code_kb=round(v * 16 / 1024, 1))
        for o in KEYS: r[o] = ops[k].get(o, 0)
        rows.append(r)
    if "--json" in sys.argv: print(json.dumps(rows, indent=1))
    else:
        print("%-70s %7s %7s " % ("kernel", "instr", "KB") + " ".join("%6s" % o for o in KEYS))
        for r in rows: print("%-70s %7d %7.1f " % (r["kernel"][:70], r["instructions"], r["code_kb"]) + " ".join("%6d" % r[o] for o in KEYS))


if __name__ == "__main__":
    main()
