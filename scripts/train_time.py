"""Times of the training ops on cuda:0 (CUDA events around repeated launches through the Python wrappers, inputs built beforehand, so
each window holds the op's own launch and kernel only), at the shapes of a 784-500-10 classifier trained on batches of 500 and at one large
OUT_PROD, with the card's name and power limit read in the same run.  Each op is timed in --windows windows; min and median are printed.
Writes nothing but stdout.

    python scripts/train_time.py [--reps N] [--windows W]
"""
import argparse
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import ggml_b200 as g  # noqa: E402

FP32_TFLOPS = 67.0       # H100 SXM data sheet, dense FP32


def time_us(fn, reps, windows):
    """(min, median) over `windows` windows of the mean time per call of `reps` calls"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            fn()
        t1.record()
        torch.cuda.synchronize()
        out.append(t0.elapsed_time(t1) * 1e3 / reps)
    out.sort()
    return out[0], out[len(out) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--windows", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"card: {q.stdout.strip()}")
    torch.manual_seed(0)
    r = lambda *s: torch.rand(s, device="cuda") * 2 - 1
    x, h, gh, go = r(500, 784), r(500, 500), r(500, 500), r(10, 500)
    logits, labels = r(500, 10), torch.nn.functional.one_hot(torch.randint(0, 10, (500,), device="cuda"), 10).float()
    w1, m1, v1 = r(500, 784), torch.zeros(500, 784, device="cuda"), torch.zeros(500, 784, device="cuda")
    params = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 0.0, 10.0, 1000.0], device="cuda")
    one = torch.ones(1, device="cuda")
    g1 = r(500, 784)
    pred, want = logits.argmax(1).int(), labels.argmax(1).int()
    rows = [
        ("OUT_PROD dW1 [784 x 500], K = 500 (grad transposed)", lambda: g.op_out_prod(x, gh.t()), 2 * 784 * 500 * 500),
        ("OUT_PROD dW2 [500 x 10], K = 500 (grad transposed)", lambda: g.op_out_prod(h, go.t()), 2 * 500 * 10 * 500),
        ("CROSS_ENTROPY_LOSS [10 x 500]", lambda: g.op_cross_entropy_loss(logits, labels), 0),
        ("CROSS_ENTROPY_LOSS_BACK [10 x 500]", lambda: g.op_cross_entropy_loss_back(one, logits, labels), 0),
        ("OPT_STEP_ADAMW [784 x 500]", lambda: g.op_opt_step_adamw(w1, g1, m1, v1, params), 0),
        ("ARGMAX [10 x 500]", lambda: g.op_argmax(logits), 0),
        ("COUNT_EQUAL [500]", lambda: g.op_count_equal(pred, want), 0),
        ("SUM [500 x 500]", lambda: g.op_sum(h), 0),
        ("REPEAT_BACK [500 x 500] -> [500]", lambda: g.op_repeat_back(h, (1, 500)), 0),
        ("STEP [500 x 500]", lambda: g.op_unary(g.UNARY_STEP, h), 0),
    ]
    print(f"{'op':56s} {'min us':>9s} {'median us':>10s}")
    for name, fn, flop in rows:
        lo, med = time_us(fn, a.reps, a.windows)
        extra = f"  {flop / med / 1e6:.2f} TFLOP/s at the median" if flop else ""
        print(f"{name:56s} {lo:9.1f} {med:10.1f}{extra}")
    A, B = r(2048, 4096), r(4096, 2048).t()
    lo, med = time_us(lambda: g.op_out_prod(A, B), 20, a.windows)
    tf = 2 * 4096 * 4096 * 2048 / med / 1e6
    print(f"{'OUT_PROD 4096 x 4096, K = 2048':56s} {lo:9.1f} {med:10.1f}  {tf:.1f} TFLOP/s = {100 * tf / FP32_TFLOPS:.0f} % of the "
          f"{FP32_TFLOPS:.0f} TFLOP/s FP32 data-sheet rate")


if __name__ == "__main__":
    main()
