"""SHA-256 of layers.sa_mlp_max's outputs on seeded inputs, at every set-abstraction level shape of
tests/test_sa_mlp_gpu.py (LEVELS) in float32, bfloat16 and float16: one JSON line per (level, dtype).

Run it in two checkouts and compare the lines to show that a change to the shared tile code (csrc/mlp_tile.cuh) leaves
the kernel's outputs bit-identical:

    python tools/sa_mlp_hashes.py --tree /path/to/checkout > hashes.jsonl
"""
import argparse
import hashlib
import json
import os
import sys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="repository checkout whose pointnet2_b200 and tests/test_sa_mlp_gpu.py are used")
    args = ap.parse_args()
    tree = os.path.abspath(args.tree)
    sys.path[:0] = [tree, os.path.join(tree, "tests")]
    import torch
    import test_sa_mlp_gpu as T
    from pointnet2_b200.layers import sa_mlp_max

    for name, n, s, k, c, widths, xyz_first, use_xyz, group_all in T.LEVELS:
        for dtype in (torch.float32, torch.bfloat16, torch.float16):
            xyz, new_xyz, points, idx = T._inputs(2, n, s, k, c, 11 + len(name), dtype)
            if group_all:
                new_xyz = idx = None
            cin = c + 3 if (use_xyz or c == 0) else c
            torch.manual_seed(5 + len(name))  # the xavier weights come from the global generator
            mlp = T._mlp(cin, widths, 5 + len(name))
            with torch.no_grad(), torch.autocast("cuda", dtype=dtype, enabled=c == 0 and dtype != torch.float32):
                got = sa_mlp_max(xyz, new_xyz, points, idx, mlp, xyz_first, use_xyz)
            digest = hashlib.sha256(got.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
            print(json.dumps({"level": name, "dtype": str(dtype).replace("torch.", ""), "sha256": digest}), flush=True)


if __name__ == "__main__":
    main()
