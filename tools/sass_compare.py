"""Compare per-kernel SASS of two libstrolle_b200.so builds: every kernel of the old build against the same kernel (for a kernel that
gained `bool NMAP` / `bool LGRID` / `bool TEXF` / `bool ENVM` / `bool LENS` template parameters: its all-<false> instantiation, whose
trailing LightGridDev, TexFilterDev, EnvMapDev and LensDev arguments are unused) of the new one.  The GI sampling kernels' ENVM is an int (EnvMode):
0 compares as false, 1 (the map) as true, 2 (the map sampled, ST_OPT_ENVIRONMENT_MAP_SAMPLING) is new.  Compared: the full instruction text (opcodes,
registers, immediates, constant-bank operands); normalised: the code-offset comments, branch targets and relocated symbol names."""
import re, subprocess, sys

def kernels(lib):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            if name: funcs[name] = body
            name, body = m.group(1), []
            continue
        if name is None: continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m:   # the instruction text without its code-offset comment; only branch targets and relocated names are normalised
            ins = m.group(1)
            if re.match(r"(@!?U?P\w+\s+)?(BRA|BSSY|CALL|JMP|JMX|BRX|BREAK|SSY|PBK|PCNT|WARPSYNC)\b", ins):
                ins = re.sub(r"0x[0-9a-f]+", "TARGET", ins)
            ins = re.sub(r"`\([^)]*\)", "SYM", ins)
            body.append(ins)
    if name: funcs[name] = body
    dem = subprocess.run(["c++filt"], input="\n".join(funcs), capture_output=True, text=True).stdout.split("\n")
    NM = ("k_prim_gbuffer", "k_gi_sampling_a", "k_ref_tracing", "k_gi_sampling_fused")                          # bool NMAP
    LG = {"k_di_sampling": 0, "k_di_sample_temporal": 0, "k_gi_sampling_b": 0, "k_ref_shading": 0, "k_gi_sampling_fused": 1}   # bool LGRID, its position
    EM = ("k_di_resolving", "k_gi_sampling_a", "k_gi_sampling_b", "k_gi_sampling_fused", "k_ref_shading")       # bool / int ENVM, the last
    def base(d):
        m = re.search(r"::(\w+)<", d)
        return m.group(1) if m and (m.group(1) in NM or m.group(1) in LG or m.group(1) in EM) else None
    def targs(d): return d.split("(")[0].split("<", 1)[1].rstrip(">").split(", ")
    def norm(d):   # the name the kernel had before it gained ENVM, TEXF, LGRID (and NMAP): all-false instantiations lose their template arguments
        k = base(d)
        if k is None: return d
        args = targs(d)
        if "LensDev)" in d:   # bool LENS (K1, K2), the last template argument
            if args[-1] == "true": return d
            del args[-1]
            head = d.split("(")[0]
            d = head.split("<")[0] + "<" + ", ".join(args) + ">" + re.sub(r", \w+::LensDev const&\)|, \w+::LensDev\)", ")", d[len(head):])
        if "EnvMapDev)" in d and args[-1] in ("0", "1", "2"):   # int ENVM: ENV_NONE / ENV_MAP as the bool it replaced
            args[-1] = {"0": "false", "1": "true", "2": "2"}[args[-1]]
            head = d.split("(")[0]
            d = head.split("<")[0] + "<" + ", ".join(args) + ">" + d[len(head):]
            if args[-1] == "2": return d
        if "EnvMapDev)" in d:   # bool ENVM, the last template argument
            if args[-1] == "true": return d
            del args[-1]
            head = d.split("(")[0]
            d = head.split("<")[0] + "<" + ", ".join(args) + ">" + re.sub(r", \w+::EnvMapDev\)", ")", d[len(head):])
            if not args: d = re.sub(r"<>", "", d, count=1)
        if "TexFilterDev)" in d:   # bool TEXF, the last template argument
            if args[-1] == "true": return d
            del args[-1]
            head = d.split("(")[0]
            d = head.split("<")[0] + "<" + ", ".join(args) + ">" + re.sub(r", \w+::TexFilterDev\)", ")", d[len(head):])
        if k in LG and len(args) > LG[k]:
            if args[LG[k]] == "true": return d
            del args[LG[k]]
            d = re.sub(r", \w+::LightGridDev\)", ")", d)
        head = d.split("(")[0]
        name = head.split("<")[0]
        if all(a == "false" for a in args): return re.sub(r"^void ", "", name) + d[len(head):]
        return name + "<" + ", ".join(args) + ">" + d[len(head):]
    return {norm(d): funcs[m] for d, m in zip(dem, funcs)}, {d for d in dem if base(d) and ({"true", "1", "2"} & set(targs(d)))}

old, _ = kernels(sys.argv[1])
new, nmap = kernels(sys.argv[2])
same = diff = 0
for k, body in sorted(old.items()):
    if k not in new: print("MISSING in new:", k); diff += 1; continue
    if new[k] == body: same += 1
    else:
        diff += 1; print(f"DIFFERS: {k}: {len(body)} vs {len(new[k])} instructions")
        if "-v" in sys.argv:
            import difflib
            print("\n".join(list(difflib.unified_diff(body, new[k], lineterm="", n=1))[:60]))
print(f"{same} kernels identical, {diff} differ; {len(old)} kernels in the old build, {len(new)} (+{len(nmap)} NMAP / LGRID / TEXF / ENVM instantiations) in the new")
for k in sorted(nmap): print("  NMAP / LGRID / TEXF / ENVM:", k)
