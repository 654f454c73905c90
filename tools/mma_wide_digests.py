"""Writes (or checks) tests/golden/mma_wide_digests.json: SHA-256 digests of the wide-tile blur pass's outputs on the
inputs of tests/mma_wide_cases.py, so a rewrite of the kernel can be held to the same bits on every sample.

    python tools/mma_wide_digests.py [--out FILE]      # write
    python tools/mma_wide_digests.py --check [FILE]    # compare, exit 1 on any difference
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import imagemagick_b200 as im  # noqa: E402
import mma_wide_cases  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "mma_wide_digests.json"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", type=Path, default=GOLDEN)
    ap.add_argument("--check", type=Path, nargs="?", const=GOLDEN)
    args = ap.parse_args()
    got = {}
    for name, kind, w, h, make in mma_wide_cases.cases():
        out, wide = mma_wide_cases.run(im, kind, make())
        assert wide >= 1, (name, wide)
        got[name] = mma_wide_cases.sha256(out)
    if args.check:
        want = json.loads(args.check.read_text())
        bad = sorted(k for k in want if got.get(k) != want[k])
        print(json.dumps({"cases": len(want), "differing": bad}))
        sys.exit(1 if bad or set(want) != set(got) else 0)
    args.out.parent.mkdir(parents=True, exist_ok=True)
    args.out.write_text(json.dumps(got, indent=1, sort_keys=True) + "\n")
    print(f"{len(got)} digests -> {args.out}")


if __name__ == "__main__":
    main()
