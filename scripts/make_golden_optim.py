"""Records the optimizer launch's bitwise goldens with the library of an earlier release:

  * tests/golden/optim_null_scaler.pt: three optimizer steps of lb_optim_step_fused and of
    lb_optim_step_dp (world 1) with no loss scaler, as the release before fp16 loss scaling computed
    them (tests/test_grad_scaler_gpu.py::test_no_scaler_is_bit_identical_to_the_previous_release);
  * tests/golden/optim_paths.pt: eight loss-scaled steps of both launches (world 1; an inf at step 2,
    a NaN at step 4) and three unscaled steps of lb_optim_step_fused at world_size 2, as the release
    before the two launches shared one kernel computed them
    (tests/test_grad_scaler_gpu.py::test_optimizer_paths_are_bit_identical_to_the_previous_release).

Each test replays the stored inputs through the current library and requires the same bits. Run on
a GPU with the previous release's package first on the path, e.g.

    git worktree add /tmp/prev 623e862 && (cd /tmp/prev && python -m lora_b200.build)
    python scripts/make_golden_optim.py --previous-release /tmp/prev --which paths

(optim_null_scaler.pt was recorded from e348b16). The inputs (the start point p0 of the test's
two-group arena and seeded host gradients) are stored with the outputs, so a golden does not depend
on device RNG."""
import argparse
import importlib.util
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--previous-release", required=True, help="checkout (built) of the release to record")
    ap.add_argument("--which", choices=("null_scaler", "paths"), default="null_scaler")
    ap.add_argument("--out", default=None, help="default: tests/golden/optim_<which>.pt")
    args = ap.parse_args()
    out_path = args.out or os.path.join(GOLD, f"optim_{args.which}.pt")
    prev = os.path.abspath(args.previous_release)
    sys.path.insert(0, prev)
    import torch
    import lora_b200
    if os.path.dirname(os.path.abspath(lora_b200.__file__)) != os.path.join(prev, "lora_b200"):
        raise SystemExit(f"lora_b200 was imported from {lora_b200.__file__}, not from {prev}")
    spec = importlib.util.spec_from_file_location("tgs", os.path.join(ROOT, "tests", "test_grad_scaler_gpu.py"))
    tgs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tgs)
    arena = tgs._two_group_arena()
    gen = torch.Generator().manual_seed(123)
    if args.which == "null_scaler":
        inputs = {"p0": arena.p.cpu().clone(),
                  "grads": [torch.randn(arena.n, generator=gen) * s for s in (0.01, 2.0, 0.01)]}
        out = {"inputs": inputs}
        for mode in ("fused", "dp"):
            out[mode] = tgs.null_scaler_run(mode, inputs)
        torch.save(out, out_path)
        print(f"wrote {out_path}: n = {arena.n}, gnorm fused {float(out['fused']['gnorm']):.6g} "
              f"dp {float(out['dp']['gnorm']):.6g}")
        return
    inputs = tgs.optim_paths_inputs(arena, gen)
    out = {"inputs": inputs}
    for run in tgs.OPTIM_PATHS:
        out[run] = tgs.optim_paths_run(run, inputs)
    torch.save(out, out_path)
    print(f"wrote {out_path}: n = {arena.n}, " + ", ".join(
        f"{run} gnorm {out[run]['gnorm'].tolist()}" for run in tgs.OPTIM_PATHS))


if __name__ == "__main__":
    main()
