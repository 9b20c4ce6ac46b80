#!/usr/bin/env python3
"""Write a checkpoint's model as a .dlw weight file for the C ABI's `delora_odometry_*` entry points
(delora_b200/deploy/export.py; byte layout in include/delora_b200.h).  The image size and fields of view come from
the checkpoint's `parameters` when it has them (they win over config/*.yaml, as in bin/run_testing.py);
`--n_stride` (max points per scan) and `--max_batch` (max pairs per delora_odometry_pairs call) size the buffers.
`--training-state` writes a .dlt training checkpoint instead (weights + Adam's state, for examples/odometry_train.c);
`--init-seed N` replaces the checkpoint by a freshly initialised model of the YAML configuration."""
import os
import sys

import click

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from delora_b200.deploy import export as export_module  # noqa: E402


@click.command()
@click.option("--checkpoint", default=None, help="Checkpoint written by the trainer (torch.save).")
@click.option("--dataset", default="kitti", show_default=True, help="Dataset whose range image the model runs on.")
@click.option("--out", required=True, help="Output .dlw file (.dlt with --training-state).")
@click.option("--n_stride", default=131072, show_default=True, help="Max points per scan.")
@click.option("--max_batch", default=1, show_default=True, help="Max pairs per delora_odometry_pairs call.")
@click.option("--config_dir", default="config", show_default=True, help="YAML files, used when the checkpoint has no "
              "`parameters`.")
@click.option("--preprocessing-normals", "preprocessing_normals", is_flag=True, default=False,
              help="Training through the C ABI estimates the normals at horizontal_cells_preprocessing and projects "
                   "the points at the model width, as the reference's preprocessing + training does (w_pre in the "
                   "header).  Off: normals at the model width.  Inference ignores it.")
@click.option("--training-state", "training_state", is_flag=True, default=False,
              help="Write a .dlt training checkpoint: the weights plus the checkpoint's Adam state (zero moments if it "
                   "has none); training resumes from it with the ICP objective, as the reference's Trainer does.")
@click.option("--init-seed", "init_seed", type=int, default=None,
              help="Instead of --checkpoint: a freshly initialised model of the YAML configuration (torch's default "
                   "initialisation, seeded), for a from-scratch start (with --training-state: in the identity "
                   "pre-training phase unless unsupervised_at_start is set).")
def main(checkpoint, dataset, out, n_stride, max_batch, config_dir, preprocessing_normals, training_state, init_seed):
    if (checkpoint is None) == (init_seed is None):
        raise click.UsageError("give exactly one of --checkpoint and --init-seed")
    d = export_module.export(checkpoint, dataset, out, n_stride, max_batch, config_dir, preprocessing_normals,
                             training_state, init_seed)
    print(f"wrote {out}: {d.H}x{d.W}, layers {list(d.layers)}, act {'relu' if d.act == 1 else 'tanh'}, "
          f"resnet_outputs {d.resnet_outputs}, single_mlp {d.single_mlp}, n_stride {d.n_stride}, max_batch {d.max_batch}"
          + (f", training normals at {d.H}x{d.w_pre}" if d.w_pre else ""))


if __name__ == "__main__":
    main()
