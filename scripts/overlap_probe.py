"""Do the FP64-bound table kernel (k_rows6) and the tensor-bound convs (k_conv_wg) actually run TOGETHER on an SM?

VERDICT r1 weak #10: "FP64 || tensor overlap is asserted, not shown".  This probe times, on one GPU,
  A  a loop of Model.infer(0) calls (in-conv + 8 dense 5x5 + 2 dense 3x3 + head; tensor pipe) alone,
  B  a loop of two-phase logistic pushes (k_rows6 + k_push_pairs; FP64 pipe) alone,
  C  both loops at once on two CUDA streams of equal priority,
  D  both at once with the convs on a high-priority stream,
and samples power and SM clock with nvidia-smi during each phase.  If the pipes overlap, C or D is close to
max(A, B) (scaled by whatever the power cap does to the clock); if the kernels merely take turns it is A + B.
Prints one JSON line.  Usage: python scripts/overlap_probe.py [streams] [iters]
"""
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bitswap_b200 import synthetic                            # noqa: E402
from bitswap_b200._lib import lib, check                     # noqa: E402
from bitswap_b200.config import preset                       # noqa: E402
from bitswap_b200.model import Model                         # noqa: E402
from bitswap_b200.streams import StreamSet                   # noqa: E402


class Smi:
    def __init__(self):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        self.p = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader,nounits", "-lms", "50"],
                                  stdout=self.f, stderr=subprocess.DEVNULL)

    def stop(self):
        self.p.terminate()
        self.p.wait(timeout=5)
        rows = [r.split(",") for r in open(self.f.name).read().strip().splitlines() if r.strip()]
        os.unlink(self.f.name)
        v = [(float(a), float(b)) for a, b in rows if a.strip().replace(".", "").isdigit()]
        if not v:
            return {}
        busy = [x for x in v if x[1] > 0.6 * max(b for _, b in v)] or v
        return {"sm_mhz_median": float(np.median([a for a, _ in busy])), "power_w_median": float(np.median([b for _, b in busy])),
                "power_w_max": max(b for _, b in v), "samples": len(v)}


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 12
    torch.cuda.set_device(0)
    cfg = preset("cifar8")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=True).load_state_dict(sd)
    m.compress()
    x = torch.from_numpy((np.random.RandomState(0).randint(0, 256, (B, cfg.xdim)) - 127.5) / 127.5).float().cuda()
    # one latent level of rows for the coder loop
    L, S, q = cfg.zdim, 1024, 10
    rs = np.random.RandomState(1)
    ends = np.linspace(-6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L), S + 1, axis=1)[:, 1:-1]
    pad = np.full((L, S), 1e300); pad[:, :S - 1] = ends
    e_pad = torch.from_numpy(pad).cuda()
    mu = torch.from_numpy(rs.normal(0, 1, (B, L)).astype(np.float32)).cuda()
    sc = torch.from_numpy(rs.uniform(0.5, 1.0, (B, L)).astype(np.float32)).cuda()
    sym = torch.from_numpy(rs.randint(0, S, (B, L)).astype(np.int16)).cuda()
    nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ss = StreamSet(B, 4096 + 64 * iters * 8 * 20)
    w, head = synthetic.initial_words(4096, seed=100)
    ss.fill(w, head)
    check(lib().bsw_set_rows_mode(1))
    s_conv_hi, s_conv, s_rows = torch.cuda.Stream(priority=-1), torch.cuda.Stream(), torch.cuda.Stream()

    def conv_loop(n, st):
        with torch.cuda.stream(st):
            for _ in range(n):
                m.infer(0)(x)

    def rows_loop(n, st):
        with torch.cuda.stream(st):
            for _ in range(n):
                check(lib().bsw_logistic_push_2p(ss.handle, 0, B, mu.data_ptr(), L, sc.data_ptr(), L, e_pad.data_ptr(), S, sym.data_ptr(),
                                                 L, S, 31, q, scratch.data_ptr(), nbytes, ctypes.c_void_p(st.cuda_stream)))

    def timed(fn):
        torch.cuda.synchronize()
        smi = Smi()
        time.sleep(0.15)
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        time.sleep(0.1)
        return dt * 1e3, smi.stop()

    nconv, nrows = iters, iters * 8                          # roughly equal device time (measured below)
    conv_loop(2, s_conv); rows_loop(4, s_rows); torch.cuda.synchronize()
    ss.fill(w, head)
    out = {"streams": B}
    out["A_conv_alone_ms"], out["A_smi"] = timed(lambda: conv_loop(nconv, s_conv))
    out["B_rows_alone_ms"], out["B_smi"] = timed(lambda: rows_loop(nrows, s_rows))
    ss.fill(w, head)
    out["C_both_equal_priority_ms"], out["C_smi"] = timed(lambda: (conv_loop(nconv, s_conv), rows_loop(nrows, s_rows)))
    ss.fill(w, head)
    out["D_both_conv_high_priority_ms"], out["D_smi"] = timed(lambda: (rows_loop(nrows, s_rows), conv_loop(nconv, s_conv_hi)))
    ss.fill(w, head)
    out["E_rows_first_then_conv_high_ms"], out["E_smi"] = timed(lambda: (rows_loop(nrows // 2, s_rows), conv_loop(nconv, s_conv_hi), rows_loop(nrows - nrows // 2, s_rows)))
    out["sum_A_B_ms"] = out["A_conv_alone_ms"] + out["B_rows_alone_ms"]
    out["max_A_B_ms"] = max(out["A_conv_alone_ms"], out["B_rows_alone_ms"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
