"""The reference's examples/train_mmoe_on_synthetic_estimator.py: MMoE on the synthetic two-task data.

Same setup: EXAMPLE_DIM = 256 numeric columns C0..C255, MMoE(num_tasks=2, num_experts=2, task_hidden_units=[32, 10],
expert_hidden_units=[64, 32]), a mean-squared-error loss per task, Adam(learning_rate=0.01), batches of 512 from
SyntheticForMultiTask(512 * 1000, example_dim=256): the first 800 batches of one input_fn call train, batches
800..999 of another call evaluate (each call draws a new dataset, as in the reference).
One Adam step is taken per batch on loss0 + loss1.  The reference groups two `minimize` calls on one optimizer with
`tf.group`, which runs them in no defined order; a single step on the summed loss is the deterministic reading.
The per-task MSE over the first and last 100 training batches and over the evaluation batches is printed.

    python examples/train_mmoe_on_synthetic_estimator.py [--train-batches N] [--eval-batches N]
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deep_recommenders_b200 import feature_column as fc  # noqa: E402
from deep_recommenders.datasets import SyntheticForMultiTask  # noqa: E402
from deep_recommenders.estimator.models.multi_task_learning import MMoE  # noqa: E402

EXAMPLE_DIM = 256


def build_columns():
    return [fc.numeric_column("C{}".format(i)) for i in range(EXAMPLE_DIM)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train-batches", type=int, default=800)
    ap.add_argument("--eval-batches", type=int, default=200)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()
    np.random.seed(args.seed)
    dev = torch.device("cuda")
    model = MMoE(build_columns(), num_tasks=2, num_experts=2, task_hidden_units=[32, 10],
                 expert_hidden_units=[64, 32], seed=args.seed, device=dev)
    opt = torch.optim.Adam(list(model.parameters()), lr=0.01, eps=1e-8)    # tf.train.AdamOptimizer defaults
    synthetic = SyntheticForMultiTask(512 * 1000, example_dim=EXAMPLE_DIM)

    def losses(features, labels):
        outputs = model(features)
        l0 = ((outputs[0] - torch.from_numpy(labels["labels0"]).to(dev).unsqueeze(1)) ** 2).mean()
        l1 = ((outputs[1] - torch.from_numpy(labels["labels1"]).to(dev).unsqueeze(1)) ** 2).mean()
        return l0, l1

    hist = []
    for step, (features, labels) in enumerate(synthetic.input_fn().take(args.train_batches)):
        l0, l1 = losses(features, labels)
        opt.zero_grad(set_to_none=True)
        (l0 + l1).backward()
        opt.step()
        hist.append(torch.stack([l0.detach(), l1.detach()]))
        if (step + 1) % 100 == 0:
            a = torch.stack(hist[-100:]).mean(0).tolist()
            print(f"step {step + 1}: task0_loss {a[0]:.4f} task1_loss {a[1]:.4f}")
    h = torch.stack(hist).cpu().numpy()
    w = min(100, len(h) // 2)
    first, last = h[:w].mean(0), h[-w:].mean(0)
    with torch.no_grad():
        ev = [torch.stack(losses(f, l)) for f, l in
              synthetic.input_fn().skip(args.train_batches).take(args.eval_batches)]
    ev = torch.stack(ev).mean(0).tolist() if ev else [float("nan")] * 2
    print(f"train mse, first {w} batches: task0 {first[0]:.4f} task1 {first[1]:.4f}")
    print(f"train mse, last {w} batches:  task0 {last[0]:.4f} task1 {last[1]:.4f}")
    print(f"eval mse ({args.eval_batches} batches of a new draw): task0 {ev[0]:.4f} task1 {ev[1]:.4f}")
    if not (last[0] < first[0] and last[1] < first[1]):
        raise SystemExit("a task loss did not fall")


if __name__ == "__main__":
    main()
