"""Odometry weight files (.dlw) for the C ABI's `delora_odometry_*` entry points (include/delora_b200.h).

A .dlw file is a 128-byte header -- magic, ABI version, the `delora_odometry_desc` fields, the blob length -- followed
by the fp32 tensors of `OdometryModel.state_dict()` concatenated in state_dict order.  A C host reads it with `fread`
alone and hands the blob to `delora_odometry_load_weights`.  The network configuration comes from the checkpoint's
`parameters` dict when it carries one (it wins over the YAML files, as in bin/run_testing.py), otherwise from
`config/*.yaml` (angles there are in degrees).  Checkpoints of models the C ABI cannot express are refused:
`pre_feature_extraction: True` and `factor_fewer_resnet_channels != 1`; dropout is the identity at inference.
`normalization_scaling: True` is recorded in the header's `model_flags` (DELORA_MODEL_NORMALIZATION_SCALING): such a
model runs through `delora_odometry_pairs_normalized`, and reading the file back restores the key.  `use_dropout: True`
is recorded as DELORA_MODEL_DROPOUT: training steps then apply the encoder's dropouts (DELORA_TRAIN_DROPOUT), inference
ignores the bit, and reading the file back restores the key.  The ICP objective the model is configured with
(`point_to_point_loss`, `point_to_plane_loss`, `plane_to_plane_loss`, `normal_loss`, `lambda_po2pl`, `po2po_alone`) is
recorded as `objective_flags` and `lambda_po2pl` (header bytes 108 and 112), so C hosts train, score and adapt on it;
files with zeros there stand for the shipped objective (point-to-plane and plane-to-plane, squared, lambda_po2pl 1).

A .dlt file is a training checkpoint for `delora_odometry_train_set_state`: a 256-byte header (the .dlw header with
its own magic, then Adam's step count, the epoch, the phase, Adam's hyperparameters, the last epoch loss and the
dropout seed) followed
by the weights, Adam's exp_avg and exp_avg_sq.  It converts both ways to the reference Trainer's checkpoint dict.
"""
import collections
import dataclasses
import os
import struct

import numpy as np
import torch

from .. import _lib

MAGIC = b"DELORAW\x00"
HEADER_BYTES = 128
# magic, abi_version, header_bytes | H, W, hfov0, hfov1, vfov0, vfov1 | n_stride, max_batch, act, layers[4],
# resnet_outputs, single_mlp, w_pre (byte 92; files written before the field have zeros there) | blob_floats |
# model_flags (byte 104; zeros in files written before the field: no flag) | objective_flags, lambda_po2pl (bytes 108,
# 112; zeros in files written before the fields: the shipped objective) | 12 reserved bytes
_HEADER = struct.Struct("<8sii" + "ii4d" + "iii4iiii" + "q" + "IIf12x")
# the shipped objective (config/hyperparameters.yaml), which objective_flags = 0 stands for
SHIPPED_OBJECTIVE = (_lib.LOSS_PO2PL | _lib.LOSS_PL2PL, 1.0)
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


def model_flags_from_config(config):
    """The header's model_flags of a configuration: DELORA_MODEL_NORMALIZATION_SCALING for normalization_scaling,
    DELORA_MODEL_DROPOUT for use_dropout."""
    flags = _lib.MODEL_NORMALIZATION_SCALING if config.get("normalization_scaling", False) else 0
    return flags | (_lib.MODEL_DROPOUT if config.get("use_dropout", False) else 0)


def objective_from_config(config):
    """-> (objective_flags, lambda_po2pl) of a configuration's ICP objective, as Deployer._flags derives the loss bits,
    plus DELORA_LOSS_PO2PO_ALONE for po2po_alone.  Missing keys take config/hyperparameters.yaml's values (the shipped
    objective).  Refused, naming the key: no loss enabled, a normal_loss other than "squared" and "linear"
    (src/losses/icp_losses.py:240), and po2po_alone with point_to_plane_loss or plane_to_plane_loss (the reference
    would read lists it never built, :135-146)."""
    po2po = bool(config.get("point_to_point_loss", False))
    po2pl = bool(config.get("point_to_plane_loss", True))
    pl2pl = bool(config.get("plane_to_plane_loss", True))
    alone = bool(config.get("po2po_alone", False))
    normal_loss = config.get("normal_loss", "squared")
    lam = float(config.get("lambda_po2pl", 1.0))
    if normal_loss not in ("squared", "linear"):
        raise ValueError(f"normal_loss: {normal_loss!r} must be 'squared' or 'linear'")
    if alone and (po2pl or pl2pl):
        raise ValueError("po2po_alone: True cannot be combined with point_to_plane_loss or plane_to_plane_loss (the "
                         "point-only objective estimates no normals)")
    if not (po2po or po2pl or pl2pl or alone):
        raise ValueError("point_to_point_loss, point_to_plane_loss, plane_to_plane_loss: no loss is enabled")
    if not np.isfinite(lam):
        raise ValueError(f"lambda_po2pl: {lam} must be finite")
    if alone:
        return _lib.LOSS_PO2PO | _lib.LOSS_PO2PO_ALONE, lam
    flags = (_lib.LOSS_PO2PO if po2po else 0) | (_lib.LOSS_PO2PL if po2pl else 0)
    if pl2pl:
        flags |= _lib.LOSS_PL2PL | (_lib.NORMAL_LINEAR if normal_loss == "linear" else 0)
    return flags, lam


def file_objective(header):
    """(objective_flags, lambda_po2pl) of a read_dlw / read_dlt header dict, the shipped objective for a file written
    before the fields (zeros there): the loss_flags ICP bits and lambda_po2pl its model trains on."""
    if header["objective_flags"] == 0:
        return SHIPPED_OBJECTIVE
    return int(header["objective_flags"]), float(header["lambda_po2pl"])


def config_objective(objective):
    """The configuration keys of an (objective_flags, lambda_po2pl) pair: the inverse of objective_from_config."""
    flags, lam = objective if objective[0] else SHIPPED_OBJECTIVE
    alone = bool(flags & _lib.LOSS_PO2PO_ALONE)
    return {"point_to_point_loss": bool(flags & _lib.LOSS_PO2PO), "point_to_plane_loss": bool(flags & _lib.LOSS_PO2PL),
            "plane_to_plane_loss": bool(flags & _lib.LOSS_PL2PL),
            "normal_loss": "linear" if flags & _lib.NORMAL_LINEAR else "squared", "lambda_po2pl": float(lam),
            "po2po_alone": alone}


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


def _pack_header(magic, header_bytes, desc, blob_floats, model_flags, objective):
    flags, lam = objective if objective is not None else (0, 0.0)
    return _HEADER.pack(magic, _lib.ABI_VERSION, header_bytes, desc.H, desc.W, desc.hfov0, desc.hfov1, desc.vfov0,
                        desc.vfov1, desc.n_stride, desc.max_batch, desc.act, *list(desc.layers), desc.resnet_outputs,
                        desc.single_mlp, desc.w_pre, blob_floats, int(model_flags), int(flags), float(lam))


def _unpack_header(raw, path, magic, what):
    """The first 128 bytes of a .dlw / .dlt file -> (header dict, desc)."""
    if len(raw) != HEADER_BYTES:
        raise ValueError(f"{path}: truncated header")
    v = _HEADER.unpack(raw)
    if v[0] != magic:
        raise ValueError(f"{path}: not an odometry {what} file (magic {v[0]!r})")
    names = ("magic", "abi_version", "header_bytes", "H", "W", "hfov0", "hfov1", "vfov0", "vfov1", "n_stride",
             "max_batch", "act", "l0", "l1", "l2", "l3", "resnet_outputs", "single_mlp", "w_pre", "blob_floats",
             "model_flags", "objective_flags", "lambda_po2pl")
    h = dict(zip(names, v))
    h["layers"] = [h.pop("l0"), h.pop("l1"), h.pop("l2"), h.pop("l3")]
    d = _lib.OdometryDesc()
    for k in ("H", "W", "hfov0", "hfov1", "vfov0", "vfov1", "n_stride", "max_batch", "act", "resnet_outputs",
              "single_mlp", "w_pre"):
        setattr(d, k, h[k])
    d.layers[:] = h["layers"]
    return h, d


def write_dlw(path, desc, blob, model_flags=0, objective=None):
    """model_flags: DELORA_MODEL_* bits (model_flags_from_config); objective: (objective_flags, lambda_po2pl)
    (objective_from_config), or None for zeros (the shipped objective)."""
    blob = np.ascontiguousarray(blob, dtype=np.float32)
    with open(path, "wb") as f:
        f.write(_pack_header(MAGIC, HEADER_BYTES, desc, blob.size, model_flags, objective))
        f.write(blob.tobytes())


def read_dlw(path):
    """-> (header dict, desc, blob float32 array); the header dict has `model_flags`, `objective_flags` and
    `lambda_po2pl` as stored (file_objective resolves zeros to the shipped objective)."""
    with open(path, "rb") as f:
        h, d = _unpack_header(f.read(HEADER_BYTES), path, MAGIC, "weight")
        blob = np.fromfile(f, dtype=np.float32)
    if blob.size != h["blob_floats"]:
        raise ValueError(f"{path}: blob has {blob.size} floats, the header says {h['blob_floats']}")
    return h, d, blob


# ---- training checkpoints (.dlt): the .dlw header and blob plus Adam's state, byte layout in include/delora_b200.h
TRAIN_MAGIC = b"DELORAT\x00"
TRAIN_HEADER_BYTES = 256
# step | epoch, unsupervised | lr, beta1, beta2, eps, loss | dropout_seed (byte 164; zeros in files written before
# the field: seed 0) | 84 zero bytes, after the 128-byte .dlw header
_TRAIN_TAIL = struct.Struct("<q" + "ii" + "5f" + "Q" + "84x")
assert HEADER_BYTES + _TRAIN_TAIL.size == TRAIN_HEADER_BYTES


@dataclasses.dataclass
class TrainingState:
    """What a .dlt file holds besides the descriptor: the fp32 weight blob, Adam's m (exp_avg) and v (exp_avg_sq) in
    blob order, the number of Adam updates, the epochs completed, the phase (unsupervised = 0: identity pre-training),
    Adam's hyperparameters, the last epoch's mean objective and the seed of the dropout masks."""
    weights: np.ndarray
    exp_avg: np.ndarray
    exp_avg_sq: np.ndarray
    step: int = 0
    epoch: int = 0
    unsupervised: int = 0
    lr: float = 1e-5
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8
    loss: float = 0.0
    dropout_seed: int = 0


def write_dlt(path, desc, state, model_flags=0, objective=None):
    """model_flags and objective as for write_dlw."""
    arrays = [np.ascontiguousarray(a, dtype=np.float32).reshape(-1)
              for a in (state.weights, state.exp_avg, state.exp_avg_sq)]
    n = arrays[0].size
    if any(a.size != n for a in arrays):
        raise ValueError(f"weights, exp_avg and exp_avg_sq must have the same length ({[a.size for a in arrays]})")
    with open(path, "wb") as f:
        f.write(_pack_header(TRAIN_MAGIC, TRAIN_HEADER_BYTES, desc, n, model_flags, objective))
        f.write(_TRAIN_TAIL.pack(int(state.step), int(state.epoch), int(state.unsupervised), state.lr, state.beta1,
                                 state.beta2, state.eps, state.loss, int(state.dropout_seed) & 0xFFFFFFFFFFFFFFFF))
        for a in arrays:
            f.write(a.tobytes())


def read_dlt(path):
    """-> (header dict, desc, TrainingState); the header dict as read_dlw's."""
    with open(path, "rb") as f:
        h, d = _unpack_header(f.read(HEADER_BYTES), path, TRAIN_MAGIC, "training")
        raw = f.read(_TRAIN_TAIL.size)
        if len(raw) != _TRAIN_TAIL.size:
            raise ValueError(f"{path}: truncated header")
        data = np.fromfile(f, dtype=np.float32)
    n = h["blob_floats"]
    if data.size != 3 * n:
        raise ValueError(f"{path}: {data.size} floats after the header, the header says 3 x {n}")
    step, epoch, unsupervised, lr, beta1, beta2, eps, loss, seed = _TRAIN_TAIL.unpack(raw)
    state = TrainingState(data[:n], data[n:2 * n], data[2 * n:], step, epoch, unsupervised, lr, beta1, beta2, eps, loss,
                          seed)
    return h, d, state


def _parameter_order(config):
    """state_dict_order, asserting that it is also the parameter order: optimizer state index i belongs to the i-th
    parameter, and OdometryModel has no BatchNorm and no other buffers."""
    from ..models.model import OdometryModel
    cfg = dict(config)
    cfg.update({"device": "cpu", "use_dropout": False})
    with torch.device("meta"):
        model = OdometryModel(cfg)
    params = [(k, tuple(v.shape)) for k, v in model.named_parameters()]
    assert not list(model.buffers()) and params == [(k, tuple(v.shape)) for k, v in model.state_dict().items()], \
        "OdometryModel has buffers: optimizer state indices no longer follow the state_dict"
    return params


def training_state_from_checkpoint(checkpoint, config):
    """The reference Trainer's checkpoint dict (src/deploy/trainer.py:155-173: model_state_dict + optimizer_state_dict
    of torch.optim.Adam) -> TrainingState.  Without optimizer state: zero moments, step 0.  A checkpoint continues with
    the ICP objective (unsupervised = 1), as the reference's Trainer does with one (:35-36).  Refused, naming the key:
    Adam settings the C step does not run (weight_decay, amsgrad, maximize), more than one parameter group,
    per-parameter steps that differ or are not integers, and tensors whose shapes do not match the model."""
    order = _parameter_order(config)
    weights = pack_state_dict(checkpoint["model_state_dict"], config)
    opt = checkpoint.get("optimizer_state_dict") or {}
    groups = opt.get("param_groups", [])
    if len(groups) > 1:
        raise ValueError(f"optimizer_state_dict.param_groups: {len(groups)} groups, the C step runs one")
    g = groups[0] if groups else {}
    for key, default in (("weight_decay", 0), ("amsgrad", False), ("maximize", False)):
        if g.get(key, default) != default:
            raise ValueError(f"optimizer_state_dict.param_groups[0].{key}: {g[key]!r} is not supported (the C step runs "
                             f"Adam with {key} = {default!r})")
    betas = g.get("betas", (0.9, 0.999))
    state = TrainingState(weights, np.zeros_like(weights), np.zeros_like(weights), 0,
                          int(checkpoint.get("epoch", -1)) + 1, 1, float(g.get("lr", config.get("learning_rate", 1e-5))),
                          float(betas[0]), float(betas[1]), float(g.get("eps", 1e-8)),
                          float(checkpoint.get("loss", 0.0)))
    per_param = opt.get("state") or {}
    if not per_param:
        return state
    ids = list(g["params"])
    if len(ids) != len(order):
        raise ValueError(f"optimizer_state_dict.param_groups[0].params: {len(ids)} parameters, the model has "
                         f"{len(order)}")
    m_parts, v_parts, steps = [], [], set()
    for pid, (key, shape) in zip(ids, order):
        s = per_param.get(pid)
        if s is None:
            raise ValueError(f"optimizer_state_dict.state[{pid}] ({key}): no state for this parameter")
        for name, parts in (("exp_avg", m_parts), ("exp_avg_sq", v_parts)):
            t = s[name]
            if tuple(t.shape) != shape:
                raise ValueError(f"optimizer_state_dict.state[{pid}].{name} ({key}): shape {tuple(t.shape)}, the "
                                 f"model needs {shape}")
            parts.append(t.detach().to("cpu", torch.float32).contiguous().reshape(-1).numpy())
        step = float(s["step"])
        if step != int(step) or step < 0:
            raise ValueError(f"optimizer_state_dict.state[{pid}].step ({key}): {step} is not a non-negative integer")
        steps.add(int(step))
    if len(steps) != 1:
        raise ValueError(f"optimizer_state_dict.state[*].step: the parameters' steps differ ({sorted(steps)[:4]}); "
                         "the C step keeps one step count")
    state.exp_avg = np.concatenate(m_parts).astype(np.float32, copy=False)
    state.exp_avg_sq = np.concatenate(v_parts).astype(np.float32, copy=False)
    state.step = steps.pop()
    return state


def checkpoint_from_training_state(state, config):
    """TrainingState -> the reference Trainer's checkpoint dict (`epoch`, `model_state_dict`, `optimizer_state_dict`,
    `loss`, `parameters`), which torch.optim.Adam.load_state_dict and both Trainers' config["checkpoint"] accept."""
    model_sd = unpack_blob(state.weights, config)
    m, v = unpack_blob(state.exp_avg, config), unpack_blob(state.exp_avg_sq, config)
    group = {k: val for k, val in torch.optim.Adam([torch.zeros(1)]).param_groups[0].items() if k != "params"}
    group.update({"lr": float(state.lr), "betas": (float(state.beta1), float(state.beta2)), "eps": float(state.eps),
                  "weight_decay": 0, "amsgrad": False, "maximize": False, "params": list(range(len(model_sd)))})
    per_param = {i: {"step": torch.tensor(float(state.step), dtype=torch.float32), "exp_avg": m[k], "exp_avg_sq": v[k]}
                 for i, k in enumerate(model_sd)}
    return {"epoch": int(state.epoch) - 1, "model_state_dict": model_sd,
            "optimizer_state_dict": {"state": per_param, "param_groups": [group]}, "loss": float(state.loss),
            "parameters": config}


def initial_training_state(config, seed):
    """A freshly initialised OdometryModel (torch's default initialisation, seeded) with a fresh Adam: the from-scratch
    start of the reference's Trainer, in the identity pre-training phase unless config["unsupervised_at_start"]."""
    from ..models.model import OdometryModel
    check_supported(config)
    cfg = dict(config)
    cfg.update({"device": "cpu", "use_dropout": False})
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(int(seed))
        model = OdometryModel(cfg)
    weights = pack_state_dict(model.state_dict(), config)
    return TrainingState(weights, np.zeros_like(weights), np.zeros_like(weights), 0, 0,
                         1 if config.get("unsupervised_at_start", False) else 0,
                         float(config.get("learning_rate", 1e-5)))


def config_from_desc(desc, base=None, dataset="kitti", model_flags=None, objective=None):
    """`base` (e.g. the YAML configuration) with the network and range-image keys set from a .dlw / .dlt descriptor,
    so that the configuration describes the weights of the file.  model_flags (the header's, or None to keep `base`'s
    values): sets normalization_scaling and use_dropout (a file without a bit means False).  objective (the header's
    (objective_flags, lambda_po2pl), or None to keep `base`'s values): sets the ICP objective's keys (config_objective;
    zeros: the shipped objective)."""
    cfg = dict(base or {})
    ds = dict(cfg.get(dataset, {}))
    ds.update({"vertical_cells": int(desc.H), "horizontal_cells": int(desc.W),
               "vertical_field_of_view": [float(desc.vfov0), float(desc.vfov1)]})
    if desc.w_pre:
        ds["horizontal_cells_preprocessing"] = int(desc.w_pre)
    cfg[dataset] = ds
    cfg.update({"horizontal_field_of_view": [float(desc.hfov0), float(desc.hfov1)],
                "activation_fct": "relu" if desc.act == 1 else "tanh", "layers": [int(v) for v in desc.layers],
                "resnet_outputs": int(desc.resnet_outputs), "use_single_mlp_at_output": bool(desc.single_mlp),
                "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1})
    if model_flags is not None:
        cfg["normalization_scaling"] = bool(int(model_flags) & _lib.MODEL_NORMALIZATION_SCALING)
        cfg["use_dropout"] = bool(int(model_flags) & _lib.MODEL_DROPOUT)
    if objective is not None:
        cfg.update(config_objective(objective))
    cfg.setdefault("use_dropout", False)
    cfg.setdefault("datasets", [dataset])
    return cfg


def export(checkpoint_path, dataset, out_path, n_stride, max_batch=1, config_dir="config", preprocessing_normals=False,
           training_state=False, init_seed=None):
    """Checkpoint (torch.save of the trainer's dict, or a bare state dict with `config_dir` YAMLs) -> .dlw file.
    training_state: write a .dlt instead (the checkpoint's optimizer state too).  init_seed (checkpoint_path None): the
    weights of a freshly initialised model of the `config_dir` YAMLs instead of a checkpoint's."""
    if init_seed is not None:
        config = model_config(None, config_dir)
        state = initial_training_state(config, init_seed)
    else:
        ckpt = torch.load(checkpoint_path, map_location="cpu", weights_only=False)
        config = model_config(ckpt, config_dir)
        if not (isinstance(ckpt, dict) and "model_state_dict" in ckpt):
            ckpt = {"model_state_dict": ckpt}
        state = training_state_from_checkpoint(ckpt, config) if training_state else None
    desc = desc_from_config(config, dataset, n_stride, max_batch, preprocessing_normals)
    flags = model_flags_from_config(config)
    objective = objective_from_config(config)
    if training_state:
        write_dlt(out_path, desc, state, flags, objective)
    else:
        write_dlw(out_path, desc, state.weights if state else pack_state_dict(ckpt["model_state_dict"], config), flags,
                  objective)
    return desc
