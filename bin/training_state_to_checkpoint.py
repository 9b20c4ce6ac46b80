#!/usr/bin/env python3
"""Turn a .dlt training checkpoint (written by examples/odometry_train.c or bin/export_odometry_weights.py
--training-state) back into the reference Trainer's checkpoint (.pth: `epoch`, `model_state_dict`,
`optimizer_state_dict`, `loss`, `parameters`), loadable by its `--checkpoint` option and by torch.optim.Adam.
`parameters` is the YAML configuration of `--config_dir` (when it exists) with the network and range-image keys of
the file's header, `normalization_scaling` and `use_dropout` from its model_flags, and the ICP objective's keys
(`point_to_point_loss`, `point_to_plane_loss`, `plane_to_plane_loss`, `normal_loss`, `lambda_po2pl`, `po2po_alone`)
from its objective fields (the shipped objective for a file with zeros there)."""
import os
import sys

import click
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from delora_b200.deploy import export as export_module  # noqa: E402


@click.command()
@click.option("--dlt", "dlt_path", required=True, help="Input .dlt file.")
@click.option("--out", required=True, help="Output checkpoint (.pth).")
@click.option("--dataset", default="kitti", show_default=True, help="Dataset whose range image the header describes.")
@click.option("--config_dir", default="config", show_default=True, help="YAML files for `parameters` (optional).")
def main(dlt_path, out, dataset, config_dir):
    header, desc, state = export_module.read_dlt(dlt_path)
    base = export_module.model_config(None, config_dir) if os.path.isdir(config_dir) else None
    config = export_module.config_from_desc(desc, base, dataset, header["model_flags"],
                                            (header["objective_flags"], header["lambda_po2pl"]))
    torch.save(export_module.checkpoint_from_training_state(state, config), out)
    print(f"wrote {out}: epoch {state.epoch - 1}, Adam step {state.step}, loss {state.loss:.9g}, "
          f"{'unsupervised' if state.unsupervised else 'identity pre-training'}")


if __name__ == "__main__":
    main()
