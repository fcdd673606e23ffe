"""Same-box A/B of library builds (machines differ by +-5 %, so builds must be compared on ONE machine, in one run).

usage:  python tools/ab.py [--conv 6 2 0] [--bench] [--batch 32] [--steps 100] -- base "CC_LIB=/path/to/other/libclearcam_b200.so" ...
Each variant ("base" = the in-tree build, or a space-separated list of VAR=value set for its process, normally CC_LIB
selecting another build) runs tools/one_conv.py on the given shapes and/or bench.py --no-cpu in a fresh process; one
table is printed at the end."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    argv = sys.argv[1:]
    if "--" not in argv:
        sys.exit(__doc__)
    opts, variants = argv[:argv.index("--")], argv[argv.index("--") + 1:]
    shapes, bench, batch, steps, i = [], False, None, None, 0
    while i < len(opts):
        if opts[i] == "--conv":
            i += 1
            while i < len(opts) and opts[i].isdigit():
                shapes.append(opts[i])
                i += 1
            continue
        if opts[i] == "--bench":
            bench = True
        elif opts[i] == "--batch":
            i += 1
            batch = opts[i]
        elif opts[i] == "--steps":     # timed steps per bench run (bench.py's default window is short for an A/B)
            i += 1
            steps = opts[i]
        i += 1
    rows = []
    for v in variants:
        env = dict(os.environ)
        if v != "base":
            env.update(kv.split("=", 1) for kv in v.split())
        row = {"variant": v}
        if shapes:
            out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "one_conv.py"), "30", *shapes], env=env, capture_output=True,
                                 text=True).stdout
            for line in out.strip().splitlines():
                shape, rest = line.split(":", 1)
                row[shape.strip()] = rest.split("ms")[0].strip() + " ms"
        if bench:
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--no-cpu", "--no-clip"] + (["--batch", batch] if batch else []) + (["--steps", steps] if steps else [])
            out = subprocess.run(cmd, env=env, capture_output=True, text=True).stdout.strip().splitlines()
            try:
                d = json.loads(out[-1])
                row["frames/s"], row["ms/step"], row["e2e"], row["frac"] = (round(d["value"], 1), round(d["ms_per_step"], 3),
                                                                             round(d["e2e"]["value"], 1), round(d["roofline"]["frac"], 4))
                row["conv TFLOP/s"] = round(d["roofline"]["achieved"], 1)
            except Exception as ex:
                row["bench"] = f"failed: {ex!r}"
        rows.append(row)
        print(row, flush=True)
    keys = []
    for r in rows:
        keys += [k for k in r if k not in keys]
    print("\n" + " | ".join(keys))
    for r in rows:
        print(" | ".join(str(r.get(k, "")) for k in keys))


if __name__ == "__main__":
    main()
