"""Encoder forward and backward on the wgmma convolution kernels.

Takes the weights of an `OdometryModel` (reference parameter names) and runs `ResNetModified._forward_impl`
(reference: src/models/resnet_modified.py:95-120, BasicBlock :159-177) through the trunk entry points of the C ABI:
`delora_trunk_forward` runs stem, max-pool, the BasicBlocks and the average pool in the launch sequence of
csrc/trunk.cu, the one the odometry entry points run as well.  `fc` and the two MLP heads (tiny GEMMs) are left to
torch, as SURVEY.md §7.6 allows.

Training (`pooled_features`, an autograd Function) keeps the activations and runs the backward as one
`delora_trunk_backward` call per stage.  Any image size the trunk takes works (ragged tiles are zero-filled / masked):
64x2048 tiles exactly, KITTI's 64x720 runs 360 -> 180 -> 90 -> 45 -> 23 wide.
"""
import ctypes

import torch

from .. import _lib, ops

_STAGE_CHANNELS = (64, 128, 256, 512)
_STAGE_STRIDES = ((1, 1), (1, 2), (1, 2), (2, 2))


class _EncoderTrainFn(torch.autograd.Function):
    """Differentiable encoder trunk on the wgmma kernels: images -> pooled [B, C4] features.  The gradients w.r.t. the
    images are not needed (the range images are data)."""

    @staticmethod
    def forward(ctx, enc, image_1, image_2, *weights):
        ctx.enc = enc
        ctx.state, pooled = enc._forward_saving(image_1, image_2)
        return pooled

    @staticmethod
    def backward(ctx, g_pooled):
        if ctx.state is None:
            raise RuntimeError("tensor-core encoder: backward called twice on the same forward (saved activations "
                               "were released); run the forward again")
        grads = ctx.enc._backward(ctx.state, g_pooled.float().contiguous())
        ctx.state[0].release()
        ctx.state = None
        if ctx.enc.grad_views is not None:
            # the kernels wrote the weight gradients into the synchroniser's flat buffer and announced them
            # (grad_ready); handing the same tensors to autograd as well would make AccumulateGrad clone each view
            # (20 device copies, 47.5 MB per step) into a p.grad that finish() replaces by the view anyway
            return (None, None, None) + (None,) * len(grads)
        return (None, None, None) + tuple(grads)


class _Slot:
    """One set of saved-activation workspaces (one per (device, B, H, W)).  A grad-enabled forward takes the lowest free
    slot and keeps it until its backward has run (or its graph is dropped), so a second forward before the first
    backward -- gradient accumulation, two model calls in one step, a loss pass interleaved with training -- never
    overwrites tensors an earlier graph still needs."""

    def __init__(self, index):
        self.index, self.busy = index, False
        self.acts = {}


class _SlotLease:
    """Held by the autograd graph of one forward; gives the slot back on backward or when the graph is dropped."""

    def __init__(self, slot):
        self.slot = slot
        slot.busy = True

    @property
    def index(self):
        return self.slot.index

    def release(self):
        self.slot.busy = False

    def __del__(self):
        self.slot.busy = False


class TensorCoreEncoder:
    def __init__(self, model):
        self.model = model
        self.act = ops.ACT_RELU if model.config["activation_fct"] == "relu" else ops.ACT_TANH
        r = model.resnet
        if r.conv1.weight.shape[0] % 64 != 0:
            raise Exception("tensor-core encoder needs channel counts that are multiples of 64 "
                            "(factor_fewer_resnet_channels = 1)")
        stages = [getattr(r, f"layer{li}") for li in range(1, 5)]
        self.layers = (ctypes.c_int * 4)(*[len(s) for s in stages])
        # trunk_parameters() indices of each stage's filters in the order its backward finishes them (last block
        # first); the stem's gradient comes with stage 0's
        self._stage_params, idx = [], 1
        for s in stages:
            per_block = []
            for blk in s:
                n = 3 if blk.downsample is not None else 2
                per_block.append(list(range(idx, idx + n)))
                idx += n
            self._stage_params.append([i for blk in reversed(per_block) for i in blk])
        self._stage_params[0].append(0)
        # bf16 weight sections, one per stem layout met (W % 2): [section, W, (versions, pointers) it was prepped from];
        # rewritten by one small kernel whenever the fp32 parameters change (every training step; after load_state_dict)
        self._weights = {}
        self._acts = {}          # inference activation workspaces by (device, B, H, W)
        self._slots = []
        # data-parallel hook (parallel_grad.BucketedGradAllReduce): weight gradients are written into these views
        # (trunk_parameters() order) and every finished stage is announced through grad_ready(list of indices)
        self.grad_views = None
        self.grad_ready = None

    def _prep(self, entry, force):
        params = self.trunk_parameters()
        version = tuple(p_._version for p_ in params) + tuple(p_.data_ptr() for p_ in params)
        if force or version != entry[2]:
            for p_ in params:
                if p_.dtype != torch.float32 or not p_.is_contiguous():
                    raise Exception("tensor-core encoder: convolution weights must be contiguous fp32")
            filters = (ctypes.c_void_p * len(params))(*[p_.data_ptr() for p_ in params])
            _lib.check(_lib.lib().delora_trunk_prep_weights(self.layers, entry[1], filters,
                                                            ops._req(entry[0], torch.uint8, "weights"), ops._stream()),
                       "delora_trunk_prep_weights")
            entry[2] = version
        return entry[0]

    def _prepped_weights(self, w, force=False):
        """-> the weight section for images w wide, up to date with the fp32 parameters."""
        dev = self.model.resnet.conv1.weight.device
        entry = self._weights.get(w % 2)
        if entry is None or entry[0].device != dev:
            n = int(_lib.lib().delora_trunk_weight_bytes(self.layers, w))
            _lib.check(int(n < 0), "delora_trunk_weight_bytes")
            entry = [torch.empty((n,), dtype=torch.uint8, device=dev), w, None]
            self._weights[w % 2] = entry
        return self._prep(entry, force)

    def _refresh_weights(self):
        """Bring every weight section up to date with the fp32 parameters (one launch each, none when unchanged)."""
        for entry in self._weights.values():
            self._prep(entry, False)

    def _workspace(self, cache, b, h, w, saving, device):
        key = (device, b, h, w)
        acts = cache.get(key)
        if acts is None:
            n = int(_lib.lib().delora_trunk_activation_bytes(self.layers, b, h, w, saving))
            _lib.check(int(n < 0), "delora_trunk_activation_bytes")
            acts = torch.zeros((n,), dtype=torch.uint8, device=device)      # halo rows stay zero forever
            cache[key] = acts
        return acts

    def _take_slot(self):
        for sl in self._slots:
            if not sl.busy:
                return _SlotLease(sl)
        sl = _Slot(len(self._slots))
        self._slots.append(sl)
        return _SlotLease(sl)

    def _trunk_forward(self, image_1, image_2, weights, acts, saving, stage_out=None):
        b, _, h, w = image_1.shape
        pooled = torch.empty((b, _STAGE_CHANNELS[-1]), dtype=torch.float32, device=image_1.device)
        _lib.check(_lib.lib().delora_trunk_forward(
            self.layers, b, h, w, self.act, saving, ops._req(image_1, torch.float32, "image_1"),
            ops._req(image_2, torch.float32, "image_2"), weights.data_ptr(), acts.data_ptr(), pooled.data_ptr(),
            stage_out, ops._stream()), "delora_trunk_forward")
        return pooled

    @torch.no_grad()
    def _infer(self, image_1, image_2):
        """-> ([x1, x2, x3, x4] as (padded NHWC bf16 view into the inference workspace, H, W), pooled [B, 512])."""
        image_1, image_2 = image_1.float().contiguous(), image_2.float().contiguous()
        b, _, h, w = image_1.shape
        weights = self._prepped_weights(w)
        acts = self._workspace(self._acts, b, h, w, 0, image_1.device)
        out = (ctypes.c_void_p * 4)()
        pooled = self._trunk_forward(image_1, image_2, weights, acts, 0, out)
        feats = []
        sh, sw = h, ops.conv_out_size(w, 2) // 2
        for s, (c, (st_h, st_w)) in enumerate(zip(_STAGE_CHANNELS, _STAGE_STRIDES)):
            sh, sw = ops.conv_out_size(sh, st_h), ops.conv_out_size(sw, st_w)
            off = out[s] - acts.data_ptr()
            n = b * (sh + 2) * (sw + 2) * c * 2
            feats.append((acts[off:off + n].view(torch.bfloat16).view(b, sh + 2, sw + 2, c), sh, sw))
        return feats, pooled

    def features(self, image_1, image_2):
        """-> [x1, x2, x3, x4] as padded NHWC bf16 + their (H, W)."""
        return self._infer(image_1, image_2)[0]

    @torch.no_grad()
    def forward(self, image_1, image_2):
        """(translation [B,3], quaternion [B,4]) like OdometryModel.forward (src/models/model.py:103-116)."""
        pooled = self._infer(image_1, image_2)[1]                                # AdaptiveAvgPool2d((1,1))
        m = self.model
        out = m.resnet.fc(pooled)
        if m.config["use_single_mlp_at_output"]:
            o = m.fully_connected_rot_trans(out)
            rot, trans = o[:, :4], o[:, 4:]
        else:
            rot, trans = m.fully_connected_rotation(out), m.fully_connected_translation(out)
        return trans, rot / torch.norm(rot)

    # ------------------------------------------------------------------------------------------
    # training path (forward keeps activations, backward runs dgrad / wgrad on the tensor cores)
    def trunk_parameters(self):
        """Conv weights in the fixed order used by the autograd function (the trunk ABI's filter order)."""
        r = self.model.resnet
        params = [r.conv1.weight]
        for li in range(1, 5):
            for blk in getattr(r, f"layer{li}"):
                params += [blk.conv1.weight, blk.conv2.weight]
                if blk.downsample is not None:
                    params.append(blk.downsample[0].weight)
        return params

    def trunk_parameter_groups(self):
        """Trunk parameter indices grouped in the order the backward finishes them: layer4, layer3, layer2,
        layer1 + stem (the last, exposed bucket is the smallest: 0.15 M parameters)."""
        return [list(self._stage_params[s]) for s in (3, 2, 1, 0)]

    def pooled_features(self, image_1, image_2):
        """[B, C4] average-pooled encoder features with autograd through the wgmma kernels."""
        return _EncoderTrainFn.apply(self, image_1.float().contiguous(), image_2.float().contiguous(),
                                     *self.trunk_parameters())

    def _forward_saving(self, image_1, image_2):
        b, _, h, w = image_1.shape
        weights = self._prepped_weights(w, force=True)          # bf16 filters of THIS step's weights
        lease = self._take_slot()
        acts = self._workspace(lease.slot.acts, b, h, w, 1, image_1.device)
        pooled = self._trunk_forward(image_1, image_2, weights, acts, 1)
        return (lease, weights, acts, (b, h, w)), pooled

    def _backward(self, state, g_pooled):
        _, weights, acts, (b, h, w) = state
        params = self.trunk_parameters()
        if self.grad_views is not None:
            grads = self.grad_views
            for g, p_ in zip(grads, params):
                if g.shape != p_.shape or g.dtype != torch.float32 or not g.is_contiguous():
                    raise ValueError(f"gradient output must be a contiguous fp32 tensor of shape {tuple(p_.shape)}")
        else:
            grads = [torch.empty_like(p_, memory_format=torch.contiguous_format) for p_ in params]
        conv_dw = (ctypes.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
        L = _lib.lib()
        for stage in (3, 2, 1, 0):
            _lib.check(L.delora_trunk_backward(self.layers, b, h, w, self.act, weights.data_ptr(), acts.data_ptr(),
                                               ops._req(g_pooled, torch.float32, "g_pooled"), conv_dw, stage,
                                               ops._stream()), "delora_trunk_backward")
            if self.grad_ready is not None:
                self.grad_ready(self._stage_params[stage])    # this stage's weight gradients are enqueued
        return grads
