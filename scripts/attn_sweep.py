"""A/B timing of the flash-attention kernel between builds of libiggt_b200.so.

  python scripts/attn_sweep.py LIB_A LIB_B [LIB ...] [--rounds 3] [--out FILE]

Every library runs in a child process of its own (IGGT_B200_LIB) and the libraries alternate, round after round, so
that clock and power drift fall on all of them alike.  A child times the C2 shapes of one GPU (frame: 8 x 1374 tokens
against themselves, global: 1 x 10992, 16 heads of 64) and the view-sharded global shapes (the local queries of one of
2 / 4 / 8 ranks against all 10992 keys) with the kv splits the library plans for them, in fp16 and bf16.  The first
round of each library also saves its outputs, and every output must equal the first library's bit for bit
(torch.equal).  Medians over the rounds and their spread (max - min) are printed per shape; PyTorch's
scaled_dot_product_attention at the frame and global shapes is timed as a yardstick."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
M = 8 * 1374


def shapes():
    out = [("frame", 8, 1374, 1374), ("global", 1, M, M)]
    for n in (2, 4, 8):
        out.append((f"global_1of{n}", 1, M // n, M))
    return out


def child(save_dir, sdpa):
    import torch
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, HERE)
    from iggt_official_b200 import ops
    from microbench import timeit
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {}
    for dt in (torch.float16, torch.bfloat16):
        tag = "fp16" if dt == torch.float16 else "bf16"
        torch.manual_seed(0)
        qkv = (torch.randn(M, 3072, device="cuda") * 1.5).to(dt)
        for name, ns, Lq, Lk in shapes():
            q, k, v = qkv[:ns * Lq, :1024], qkv[:ns * Lk, 1024:2048], qkv[:ns * Lk, 2048:]
            out = torch.empty(ns * Lq, 1024, device="cuda", dtype=dt)
            splits = ops.attention_plan(ns, Lq, Lk, 16)[0]
            ms = timeit(lambda: ops.attention(q, k, v, ns, Lq, Lk, 16, out=out), reps=20, flush=flush)
            res[f"{name}_{tag}"] = {"ms": ms, "splits": splits,
                                    "tflops": 4.0 * ns * Lq * Lk * 1024 / ms / 1e9}
            if save_dir:
                torch.save(out.cpu(), os.path.join(save_dir, f"{name}_{tag}.pt"))
        if sdpa:
            for name, ns, L in [("frame", 8, 1374), ("global", 1, M)]:
                q4, k4, v4 = (qkv[:, 1024 * i:1024 * (i + 1)].view(ns, L, 16, 64).transpose(1, 2) for i in range(3))
                ms = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(q4, k4, v4), reps=20, flush=flush)
                res[f"sdpa_{name}_{tag}"] = {"ms": ms, "tflops": 4.0 * ns * L * L * 1024 / ms / 1e9}
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="JSON file for every round's timings and the comparison")
    a = ap.parse_args()
    if len(a.libs) < 2:
        ap.error("give at least two library paths")
    libs = [os.path.abspath(p) for p in a.libs]
    for p in libs:
        if not os.path.isfile(p):
            ap.error(f"no library at {p}")
    tmp = tempfile.mkdtemp(prefix="attn_ab_")
    runs = {i: [] for i in range(len(libs))}
    for r in range(a.rounds):
        for i, lib in enumerate(libs):
            save = os.path.join(tmp, str(i)) if r == 0 else ""
            if save:
                os.makedirs(save)
            env = dict(os.environ, IGGT_B200_LIB=lib)
            cmd = [sys.executable, os.path.abspath(__file__), "--child", save, "1" if r == 0 and i == 0 else "0"]
            p = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=HERE, timeout=900)
            lines = p.stdout.strip().splitlines()
            if p.returncode != 0 or not lines:
                sys.exit(f"library {i} ({lib}) round {r} failed:\n{p.stderr[-2000:]}")
            runs[i].append(json.loads(lines[-1]))
            print(f"round {r} lib {i} done", flush=True)

    import torch
    same = True
    equal = {}
    for i in range(1, len(libs)):
        for f in sorted(os.listdir(os.path.join(tmp, "0"))):
            x = torch.load(os.path.join(tmp, "0", f))
            y = torch.load(os.path.join(tmp, str(i), f))
            eq = torch.equal(x, y)
            equal[f"{i}:{f[:-3]}"] = eq
            same &= eq
            if not eq:
                d = (x.float() - y.float()).abs()
                print(f"lib {i} {f[:-3]}: NOT bit-identical to lib 0 (differing elements {int((d != 0).sum())}, "
                      f"max |diff| {d.max().item():.3e})")
    summary = {}
    print(f"{'shape':<22}" + "".join(f"{'lib ' + str(i) + ' ms (spread)':>26}" for i in range(len(libs))) +
          f"{'lib 1 / lib 0':>15}")
    for key in runs[0][0]:
        row = {}
        for i in range(len(libs)):
            if key not in runs[i][0]:
                continue
            t = sorted(run[key]["ms"] for run in runs[i] if key in run)
            row[i] = {"median_ms": t[len(t) // 2], "spread_ms": t[-1] - t[0],
                      "tflops": runs[i][0][key]["tflops"], "splits": runs[i][0][key].get("splits")}
        summary[key] = row
        cells = "".join(f"{row[i]['median_ms']:>16.3f} ({row[i]['spread_ms']:.3f})" if i in row else f"{'':>26}"
                        for i in range(len(libs)))
        ratio = f"{row[1]['median_ms'] / row[0]['median_ms']:>15.3f}" if 1 in row else ""
        print(f"{key:<22}{cells}{ratio}")
    print("outputs bit-identical to lib 0:", same)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"libs": libs, "rounds": runs, "summary": summary, "equal": equal, "bit_identical": same}, fh,
                      indent=1)
    shutil.rmtree(tmp)
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        child(sys.argv[2], sys.argv[3] == "1")
    else:
        main()
