"""Odometry weight files (.dlw) for the C ABI's `delora_odometry_*` entry points (include/delora_b200.h).

A .dlw file is a 128-byte header -- magic, ABI version, the `delora_odometry_desc` fields, the blob length -- followed
by the fp32 tensors of `OdometryModel.state_dict()` concatenated in state_dict order.  A C host reads it with `fread`
alone and hands the blob to `delora_odometry_load_weights`.  The network configuration comes from the checkpoint's
`parameters` dict when it carries one (it wins over the YAML files, as in bin/run_testing.py), otherwise from
`config/*.yaml` (angles there are in degrees).  Checkpoints of models the C ABI cannot express are refused:
`pre_feature_extraction: True` and `factor_fewer_resnet_channels != 1`; dropout is the identity at inference.
"""
import collections
import os
import struct

import numpy as np
import torch

from .. import _lib

MAGIC = b"DELORAW\x00"
HEADER_BYTES = 128
# magic, abi_version, header_bytes | H, W, hfov0, hfov1, vfov0, vfov1 | n_stride, max_batch, act, layers[4],
# resnet_outputs, single_mlp, w_pre (byte 92; files written before the field have zeros there) | blob_floats |
# 24 reserved bytes
_HEADER = struct.Struct("<8sii" + "ii4d" + "iii4iiii" + "q" + "24x")
assert _HEADER.size == HEADER_BYTES


def model_config(checkpoint, config_dir="config"):
    """The network configuration of a loaded checkpoint dict: its `parameters` (radians already) or the YAML files."""
    if isinstance(checkpoint, dict) and "parameters" in checkpoint:
        return dict(checkpoint["parameters"])
    import yaml
    config = {}
    for name in ("config_datasets.yaml", "deployment_options.yaml", "hyperparameters.yaml"):
        with open(os.path.join(config_dir, name)) as f:
            config.update(yaml.load(f, Loader=yaml.FullLoader))
    for ds in config["datasets"]:
        config[ds]["vertical_field_of_view"] = [a * (np.pi / 180.0) for a in config[ds]["vertical_field_of_view"]]
    config["horizontal_field_of_view"] = [a * (np.pi / 180.0) for a in config["horizontal_field_of_view"]]
    return config


def check_supported(config):
    """Raise for configurations the descriptor cannot express; the message names the key."""
    if config.get("pre_feature_extraction", False):
        raise ValueError("pre_feature_extraction: True is not supported by the odometry C ABI (the descriptor has no "
                         "pre-feature extractor)")
    if config.get("factor_fewer_resnet_channels", 1) != 1:
        raise ValueError(f"factor_fewer_resnet_channels: {config['factor_fewer_resnet_channels']} is not supported by "
                         "the odometry C ABI (only the full-width encoder, 1)")
    if config.get("activation_fct") not in ("relu", "tanh"):
        raise ValueError(f"activation_fct: {config.get('activation_fct')!r} must be 'relu' or 'tanh'")


def desc_from_config(config, dataset, n_stride, max_batch=1, preprocessing_normals=False):
    """-> _lib.OdometryDesc for the model of `config` on `dataset`'s range image.
    preprocessing_normals: train through the C ABI on the reference's recipe, normals estimated at
    `horizontal_cells_preprocessing` (w_pre); otherwise at the model width (w_pre = 0)."""
    check_supported(config)
    ds = config[dataset]
    layers = [int(v) for v in config["layers"]]
    if len(layers) != 4:
        raise ValueError(f"layers: {layers} must have 4 entries")
    hf, vf = config["horizontal_field_of_view"], ds["vertical_field_of_view"]
    d = _lib.OdometryDesc()
    d.H, d.W = int(ds["vertical_cells"]), int(ds["horizontal_cells"])
    d.hfov0, d.hfov1, d.vfov0, d.vfov1 = float(hf[0]), float(hf[1]), float(vf[0]), float(vf[1])
    d.n_stride, d.max_batch = int(n_stride), int(max_batch)
    d.act = 1 if config["activation_fct"] == "relu" else 2
    d.layers[:] = layers
    d.resnet_outputs = int(config["resnet_outputs"])
    d.single_mlp = 1 if config["use_single_mlp_at_output"] else 0
    if preprocessing_normals:
        if "horizontal_cells_preprocessing" not in ds:
            raise ValueError(f"{dataset}: horizontal_cells_preprocessing is needed for preprocessing_normals")
        d.w_pre = int(ds["horizontal_cells_preprocessing"])
    return d


def state_dict_order(config):
    """[(key, shape)] of OdometryModel(config).state_dict(), built on the meta device (no memory, no init cost)."""
    from ..models.model import OdometryModel
    cfg = dict(config)
    cfg.update({"device": "cpu", "use_dropout": False})
    with torch.device("meta"):
        model = OdometryModel(cfg)
    return [(k, tuple(v.shape)) for k, v in model.state_dict().items()]


def pack_state_dict(state_dict, config):
    """The weight blob: fp32 tensors of the state dict concatenated in OdometryModel's state_dict order."""
    check_supported(config)
    order = state_dict_order(config)
    expected = {k for k, _ in order}
    extra = sorted(set(state_dict) - expected)
    if extra:
        raise ValueError(f"state dict has keys the odometry C ABI does not use: {extra[:4]}")
    parts = []
    for key, shape in order:
        if key not in state_dict:
            raise ValueError(f"state dict lacks {key}")
        t = state_dict[key]
        if tuple(t.shape) != shape:
            raise ValueError(f"{key}: shape {tuple(t.shape)}, the configuration needs {shape}")
        parts.append(t.detach().to("cpu", torch.float32).contiguous().reshape(-1).numpy())
    return np.concatenate(parts).astype(np.float32, copy=False)


def unpack_blob(blob, config):
    """The inverse of pack_state_dict: a weight blob (e.g. read from a fine-tuned .dlw) -> an OdometryModel state dict
    of fp32 CPU tensors, loadable with `model.load_state_dict`."""
    check_supported(config)
    flat = torch.as_tensor(np.ascontiguousarray(blob, dtype=np.float32)).reshape(-1)
    order = state_dict_order(config)
    want = sum(int(np.prod(shape, dtype=np.int64)) for _, shape in order)
    if flat.numel() != want:
        raise ValueError(f"blob has {flat.numel()} floats, the configuration needs {want}")
    state, off = collections.OrderedDict(), 0
    for key, shape in order:
        n = int(np.prod(shape, dtype=np.int64))
        state[key] = flat[off:off + n].reshape(shape).clone()
        off += n
    return state


def write_dlw(path, desc, blob):
    blob = np.ascontiguousarray(blob, dtype=np.float32)
    header = _HEADER.pack(MAGIC, _lib.ABI_VERSION, HEADER_BYTES, desc.H, desc.W, desc.hfov0, desc.hfov1, desc.vfov0,
                          desc.vfov1, desc.n_stride, desc.max_batch, desc.act, *list(desc.layers), desc.resnet_outputs,
                          desc.single_mlp, desc.w_pre, blob.size)
    with open(path, "wb") as f:
        f.write(header)
        f.write(blob.tobytes())


def read_dlw(path):
    """-> (header dict, desc, blob float32 array)."""
    with open(path, "rb") as f:
        raw = f.read(HEADER_BYTES)
        if len(raw) != HEADER_BYTES:
            raise ValueError(f"{path}: truncated header")
        v = _HEADER.unpack(raw)
        if v[0] != MAGIC:
            raise ValueError(f"{path}: not an odometry weight file (magic {v[0]!r})")
        blob = np.fromfile(f, dtype=np.float32)
    names = ("magic", "abi_version", "header_bytes", "H", "W", "hfov0", "hfov1", "vfov0", "vfov1", "n_stride",
             "max_batch", "act", "l0", "l1", "l2", "l3", "resnet_outputs", "single_mlp", "w_pre", "blob_floats")
    h = dict(zip(names, v))
    h["layers"] = [h.pop("l0"), h.pop("l1"), h.pop("l2"), h.pop("l3")]
    if blob.size != h["blob_floats"]:
        raise ValueError(f"{path}: blob has {blob.size} floats, the header says {h['blob_floats']}")
    d = _lib.OdometryDesc()
    for k in ("H", "W", "hfov0", "hfov1", "vfov0", "vfov1", "n_stride", "max_batch", "act", "resnet_outputs",
              "single_mlp", "w_pre"):
        setattr(d, k, h[k])
    d.layers[:] = h["layers"]
    return h, d, blob


def export(checkpoint_path, dataset, out_path, n_stride, max_batch=1, config_dir="config", preprocessing_normals=False):
    """Checkpoint (torch.save of the trainer's dict, or a bare state dict with `config_dir` YAMLs) -> .dlw file."""
    ckpt = torch.load(checkpoint_path, map_location="cpu", weights_only=False)
    config = model_config(ckpt, config_dir)
    state = ckpt["model_state_dict"] if isinstance(ckpt, dict) and "model_state_dict" in ckpt else ckpt
    desc = desc_from_config(config, dataset, n_stride, max_batch, preprocessing_normals)
    write_dlw(out_path, desc, pack_state_dict(state, config))
    return desc
