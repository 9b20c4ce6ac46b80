"""One pass over every kernel family at 16x180 for compute-sanitizer (memcheck / racecheck / initcheck):
projection (atomicMin scatter + resolve), normals (smem halo tile), lists, sort, list ICP, dense ICP (work list +
block search), quaternion kernels, and -- unless `noenc` is given -- the tensor-core encoder forward + backward."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from delora_b200 import ops, synthetic  # noqa: E402
from delora_b200.pipeline import ScanPairPipeline  # noqa: E402

vf = (-15.0, 15.0)
h, w = 16, 180
cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vf, device="cuda")
hf, vfr = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
s1, s2, _, t_pred = synthetic.make_pair(0, w_raw=192, rings=16, vfov_deg=vf)
pipe = ScanPairPipeline(2, max(s1.shape[1], s2.shape[1]) + 5, h, w, hf, vfr, device="cuda")
pipe.load([s1, s2], [s2, s1], torch.stack((t_pred, t_pred)))
for _ in range(2):
    losses, grad_t = pipe.step()
pts = torch.zeros((2, 3, max(s1.shape[1], s2.shape[1])), device="cuda")
pts[0, :, :s1.shape[1]] = s1.cuda()
pts[1, :, :s2.shape[1]] = s2.cuda()
n = torch.tensor([s1.shape[1], s2.shape[1]], dtype=torch.int32, device="cuda")
image, imap = ops.project(pts, n, h, w, hf, vfr)
u, v, r = ops.project_uv(pts, n, h, w, hf, vfr)
order = ops.sort_by_range(r, n)
nrm = ops.normals(image)
p4, n4, cs, cnt = ops.lists_from_images(image, nrm)
T = t_pred[:3, :].reshape(1, 12).contiguous().cuda()
ops.icp_fwd_bwd(p4[1:2].contiguous(), n4[1:2].contiguous(), cnt[1:2].contiguous(), T, p4[0:1].contiguous(),
                n4[0:1].contiguous(), cs[0:1].contiguous(), h, w, hf, vfr, pointwise=True)
# grids at 16 x 200 re-projected at 16 x 180 (delora_project_grids_fwd: scatter + resolve)
_, _, pg200, ng200 = ops.project_normals(pts, n, h, 200, hf, vfr)
ops.project_grids(pg200, ng200, h, 200, w, hf, vfr)
q = torch.randn(4, 4, device="cuda")
ops.quat_to_T_bwd(q, torch.randn(4, 16, device="cuda"))
torch.cuda.synchronize()
print("geometry kernels done", float(losses[0, 1]), float(losses[0, 2]))
if "noenc" not in sys.argv:
    from delora_b200.models.model import OdometryModel
    ecfg = synthetic.fov_config(h=16, w=256, vfov_deg=vf, device="cuda")
    ecfg.update({"pre_feature_extraction": False, "resnet_outputs": 1000, "use_dropout": False, "layers": [2, 2, 2, 2],
                 "factor_fewer_resnet_channels": 1, "activation_fct": "tanh", "use_single_mlp_at_output": False})
    torch.manual_seed(0)
    model = OdometryModel(ecfg).cuda()
    img1 = torch.randn(1, 4, 16, 256, device="cuda") * 5
    img2 = torch.randn(1, 4, 16, 256, device="cuda") * 5
    t, qq = model(image_1=img1, image_2=img2)
    (t.sum() + qq.sum()).backward()
    torch.cuda.synchronize()
    print("encoder forward + backward done", float(t.abs().sum()))
# peer-memory gradient all-reduce kernel, one-rank form (flags, vector loop, tail): the multi-rank protocol needs
# concurrently resident kernels, which the sanitizer's serialisation does not give (tests/test_gpu_allreduce.py)
import ctypes  # noqa: E402
from delora_b200 import _lib  # noqa: E402
L = _lib.lib()
buf = torch.randn(5000 * 4, device="cuda")
want = buf.clone() * 0.5
flags = torch.zeros(L.delora_grad_allreduce_flag_words(), dtype=torch.int32, device="cuda")
status = torch.zeros(1, dtype=torch.int32, device="cuda")
u64 = ctypes.c_uint64 * 1
_lib.check(L.delora_grad_allreduce_f32(u64(buf.data_ptr()), u64(flags.data_ptr()), 0, 0, 1, 0, buf.numel(), 0.5, 1, 3, 64,
                                       status.data_ptr(), None), "grad_allreduce")
torch.cuda.synchronize()
assert torch.equal(buf, want) and int(status.item()) == 0
print("grad all-reduce (one rank) done")
