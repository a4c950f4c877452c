"""Record what nv_sample_topk returns on fixed score rows: the drawn ids and a SHA-256 of the fp32 distribution it draws from
(probs_out), per (temperature, top_k) case.  Recorded with the library of the commit before top-p was added to the sampler,
so tests/test_sampling_multi_gpu.py can show that nv_sample_topk, and nv_sample at top_p = 1, still return those bits.

    python tests/golden/make_sample_topk_golden.py --lib path/to/libnavillm_b200.so [--out tests/golden/sample_topk.json]

Needs a CUDA device.  Calls the C ABI through ctypes, so any build of the library can be recorded.
"""
import argparse
import ctypes
import hashlib
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from tests.test_top_p_cpu import SPECIAL, V, score_rows  # noqa: E402

CASES = [(1.0, 50), (0.6, 0), (1.3, 5), (0.7, 50), (1.0, 1)]
B = 8


def inputs():
    scores = score_rows(B, seed=7)
    u = torch.rand(B, generator=torch.Generator().manual_seed(1))
    return scores, u


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def run(fn, scores, u, temperature, top_k, dev):
    """fn(logits, ld, V, special, n_special, finished, eos, pad, stop, temperature, top_k, u, next, probs_out, B, stream)."""
    lg = scores.to(dev)
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=dev)
    fin = torch.zeros(B, dtype=torch.int32, device=dev)
    nxt = torch.full((B,), -1, dtype=torch.int32, device=dev)
    probs = torch.empty(B, V, dtype=torch.float32, device=dev)
    ud = u.to(dev)
    fn(lg, special, fin, nxt, probs, ud, temperature, top_k)
    torch.cuda.synchronize()
    return nxt.cpu().tolist(), sha(probs.cpu())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", required=True)
    ap.add_argument("--out", default=str(ROOT / "tests" / "golden" / "sample_topk.json"))
    a = ap.parse_args()
    lib = ctypes.CDLL(a.lib)
    dev = torch.device("cuda:0")
    p = lambda t: ctypes.c_void_p(t.data_ptr())

    def fn(lg, special, fin, nxt, probs, ud, temperature, top_k):
        rc = lib.nv_sample_topk(p(lg), ctypes.c_int64(lg.stride(0)), ctypes.c_int(V), p(special), ctypes.c_int(special.numel()),
                                p(fin), ctypes.c_int(2), ctypes.c_int(0), ctypes.c_int(1), ctypes.c_float(temperature),
                                ctypes.c_int(top_k), p(ud), p(nxt), p(probs), ctypes.c_int(B),
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, rc

    scores, u = inputs()
    out = {"scores_sha256": sha(scores), "u_sha256": sha(u), "cases": []}
    for temperature, top_k in CASES:
        ids, h = run(fn, scores, u, temperature, top_k, dev)
        out["cases"].append({"temperature": temperature, "top_k": top_k, "next": ids, "probs_sha256": h})
    Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
