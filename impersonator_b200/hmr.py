"""``HumanModelRecovery`` (networks/hmr.py:255-330) on this library's kernels: image -> theta (85) -> SMPL details.

Same module tree and ``state_dict`` keys as the reference (``resnet.conv1 / layer{1..4}.{i}.{bn1,conv1,bn2,conv2,bn3,conv3,
shortcut.0} / post_bn``, ``regressor.mean_theta / fc_blocks.fc{1,2,3}``, ``smpl.*``), so ``hmr.load_state_dict(torch.load(
opt.hmr_model))`` (models/imitator.py:69-74) works unchanged.  The ``nn.Conv2d`` / ``nn.BatchNorm2d`` / ``nn.Linear``
children are parameter holders; ``forward`` drives

  conv1 7x7 s2 (3 -> 64, bias)                         lwb_conv2d_direct_nchw      networks/hmr.py:124,275
  max_pool2d(3, 2, ceil_mode=True)                     lwb_maxpool_nchw_to_nhwc    :150,279
  16 pre-activation bottlenecks (1x1 / 3x3 / 1x1)      the wgmma conv engine (lwb_conv_plan_*), eval-mode BatchNorm folded
                                                       into lwb_norm_act_nhwc's per-channel affine (+ ReLU, + shortcut add,
                                                       + the NEXT block's bn1 + ReLU as the operand "post" affine)   :66-116
  relu(post_bn) + avg_pool2d(7)                        lwb_global_avgpool_nhwc     :160-163,289-292
  3 x (fc1 + ReLU, fc2 + ReLU, fc3; theta += .)        lwb_linear                  :244-252 (Dropout is the identity in eval)

``get_details(theta)`` (:302-330) goes through the SMPL LBS kernels (impersonator_b200.smpl).  Inference only (BatchNorm
uses its running statistics: the reference always calls ``hmr.eval()``).
"""
from collections import OrderedDict

import torch
import torch.nn as nn

from . import kernels as K
from ._lib import LwbError
from .binding import Operands, PlanBinder, StreamOwner, bn_affine, lo_format, split_mode, stream_for
from .smpl import SMPL


class PreActBottleneck(nn.Module):
    """networks/hmr.py:66-116 (parameter holder)."""
    expansion = 4

    def __init__(self, in_planes, planes, stride=1):
        super(PreActBottleneck, self).__init__()
        self.bn1 = nn.BatchNorm2d(in_planes)
        self.conv1 = nn.Conv2d(in_planes, planes, kernel_size=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, self.expansion * planes, kernel_size=1, bias=True)
        self.stride = stride
        if in_planes != self.expansion * planes:
            self.shortcut = nn.Sequential(nn.Conv2d(in_planes, self.expansion * planes, kernel_size=1, stride=stride, bias=True))

    def forward(self, x):
        raise LwbError("PreActBottleneck runs only inside HumanModelRecovery.forward")


class PreActResNet(nn.Module):
    """networks/hmr.py:119-166 (parameter holder; note the stride sits on the LAST block of layers 1-3, :142-146)."""

    def __init__(self, block, num_blocks):
        super(PreActResNet, self).__init__()
        self.in_planes = 64
        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=True)
        self.layer1 = self._make_layer(block, 64, num_blocks[0], stride=2)
        self.layer2 = self._make_layer(block, 128, num_blocks[1], stride=2)
        self.layer3 = self._make_layer(block, 256, num_blocks[2], stride=2)
        self.layer4 = self._make_layer(block, 512, num_blocks[3], stride=1)
        self.post_bn = nn.BatchNorm2d(2048)

    def _make_layer(self, block, planes, num_blocks, stride):
        layers = [block(self.in_planes, planes, 1)]
        self.in_planes = planes * block.expansion
        for i in range(1, num_blocks):
            layers.append(block(self.in_planes, planes, stride=stride if i == num_blocks - 1 else 1))
        return nn.Sequential(*layers)

    def blocks(self):
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            for blk in layer:
                yield blk

    def forward(self, x):
        raise LwbError("PreActResNet runs only inside HumanModelRecovery.forward")


def preActResNet50():
    return PreActResNet(PreActBottleneck, [3, 4, 6, 3])


class ThetaRegressor(nn.Module):
    """networks/hmr.py:214-252 (parameter holder; the iteration runs in HumanModelRecovery.forward)."""

    def __init__(self, input_dim, out_dim, iterations=3):
        super(ThetaRegressor, self).__init__()
        self.iterations = iterations
        self.register_buffer('mean_theta', torch.rand(out_dim, dtype=torch.float32))
        fc_blocks = OrderedDict()
        fc_blocks['fc1'] = nn.Linear(input_dim, 1024, bias=True)
        fc_blocks['relu1'] = nn.ReLU()
        fc_blocks['dropout1'] = nn.Dropout(p=0.5)
        fc_blocks['fc2'] = nn.Linear(1024, 1024, bias=True)
        fc_blocks['relu2'] = nn.ReLU()
        fc_blocks['dropout2'] = nn.Dropout(p=0.5)
        fc_blocks['fc3'] = nn.Linear(1024, out_dim, bias=True)
        nn.init.xavier_normal_(fc_blocks['fc3'].weight, gain=0.1)
        nn.init.zeros_(fc_blocks['fc3'].bias)
        self.fc_blocks = nn.Sequential(fc_blocks)


def _bn_fold(bn):
    return bn_affine(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)


class _HmrStream(object):
    """The encoder bound to (batch, 224 x 224, precision): persistent activations, conv plans, folded BatchNorms."""

    def __init__(self, net, B, dev, split):
        self.B, self.dev, self.split = B, dev, split
        self.lo_format = lo_format(split)
        r = net.resnet
        self.w1 = r.conv1.weight.detach().float().contiguous()
        self.b1 = r.conv1.bias.detach().float().contiguous()
        blocks = list(r.blocks())
        h = w = 56                                           # 224 -> conv1 s2 -> 112 -> max_pool(3, 2, ceil) -> 56
        self.x0 = torch.empty((B, h, w, 64), dtype=torch.float32, device=dev)
        pre = Operands((B, h, w, 64), dev, split)            # relu(bn1(x)) of the first block
        self.pre0 = pre
        self.pre0_ss = _bn_fold(blocks[0].bn1)
        x_f32 = self.x0
        self.steps = []
        plans = PlanBinder(dev, split)
        cmax = 2048

        for bi, blk in enumerate(blocks):
            planes = blk.conv1.weight.shape[0]
            s = blk.stride
            ho, wo = h // s, w // s
            nxt = blocks[bi + 1] if bi + 1 < len(blocks) else None
            st = dict(stride=s)
            st["c1"] = plans.conv(blk.conv1.weight.detach(), pre.pair, B, h, w, share="main")
            a1 = Operands((B, h, w, planes), dev, split)
            st["a1"], st["ss2"] = a1, _bn_fold(blk.bn2)
            st["c2"] = plans.conv(blk.conv2.weight.detach(), a1.pair, B, h, w, stride=s, share="main")
            a2 = Operands((B, ho, wo, planes), dev, split)
            st["a2"], st["ss3"] = a2, _bn_fold(blk.bn3)
            st["c3"] = plans.conv(blk.conv3.weight.detach(), a2.pair, B, ho, wo, share="main")
            bias = blk.conv3.bias.detach().float()
            if hasattr(blk, 'shortcut'):
                sc = blk.shortcut[0]
                rec = plans.conv(sc.weight.detach(), pre.pair, B, h, w, stride=s, share="shortcut")    # lives next to conv3's output
                st["sc"] = rec
                bias = bias + sc.bias.detach().float()
                st["res"], st["res_step"] = rec.out, 1
            else:
                st["sc"] = None
                st["res"], st["res_step"] = x_f32, s           # identity, subsampled by the block's stride (hmr.py:21-36,103)
            st["bias"] = bias.contiguous()
            st["out"] = torch.empty((B, ho, wo, 4 * planes), dtype=torch.float32, device=dev)
            if nxt is not None:
                st["post"] = _bn_fold(nxt.bn1)
                pre = Operands((B, ho, wo, 4 * planes), dev, split)
                st["pre"] = pre
            else:
                st["post"], st["pre"] = None, None
            x_f32 = st["out"]
            h, w = ho, wo
            self.steps.append(st)
        self.final = x_f32
        self.post_ss = _bn_fold(r.post_bn)
        plans.finalize()
        self.ws = torch.empty((B, cmax, 2), dtype=torch.float32, device=dev)
        self.range_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        reg = net.regressor
        self.fc = [(m.weight.detach().float().contiguous(), m.bias.detach().float().contiguous())
                   for m in (reg.fc_blocks.fc1, reg.fc_blocks.fc2, reg.fc_blocks.fc3)]
        self.mean_theta = reg.mean_theta.detach().float()
        self.iterations = reg.iterations
        fdim = self.fc[0][0].shape[1] - self.mean_theta.shape[0]
        if fdim != 2048:
            raise LwbError("the regressor expects %d encoder features, the encoder emits 2048" % fdim)
        self.total = torch.empty((B, self.fc[0][0].shape[1]), dtype=torch.float32, device=dev)       # [features | theta]
        self.h1 = torch.empty((B, 1024), dtype=torch.float32, device=dev)
        self.h2 = torch.empty((B, 1024), dtype=torch.float32, device=dev)

    def _affine(self, raw, ss, out, relu=True, **kw):
        K.norm_act_nhwc(raw, None, ss[0], ss[1], relu, self.ws, y_f32=kw.pop("y_f32", None), y_hi=out.hi if out is not None else None,
                        y_lo=out.lo if out is not None else None, lo_format=self.lo_format, range_flag=self.range_flag, **kw)

    def run(self, x):
        B = self.B
        if tuple(x.shape) != (B, 3, 224, 224):
            raise LwbError("HMR expects [%d,3,224,224] images in [-1,1], got %s" % (B, tuple(x.shape)))
        self.range_flag.zero_()
        c1 = K.conv2d_direct_nchw(x.float().contiguous(), self.w1, self.b1, stride=2, pad=3)           # hmr.py:275
        K.maxpool_nchw_to_nhwc(c1, 3, 2, out=self.x0)                                                    # :279
        self._affine(self.x0, self.pre0_ss, self.pre0)                                                  # relu(bn1(x)) of layer1.0
        for st in self.steps:
            if st["sc"] is not None:
                st["sc"].plan.run()                                                                     # shortcut(preact)   :101
            st["c1"].plan.run()
            self._affine(st["c1"].out, st["ss2"], st["a1"])                                             # relu(bn2(conv1))   :102
            st["c2"].plan.run()
            self._affine(st["c2"].out, st["ss3"], st["a2"])                                             # relu(bn3(conv2))   :103
            st["c3"].plan.run()
            # out = conv3 + bias (+ shortcut bias) + shortcut; operands of the next block = relu(bn1_next(out))     :104-105
            post = st["post"]
            K.norm_act_nhwc(st["c3"].out, None, None, st["bias"], False, self.ws, residual=st["res"], res_step=st["res_step"],
                            y_f32=st["out"], y_hi=st["pre"].hi if st["pre"] is not None else None,
                            y_lo=st["pre"].lo if st["pre"] is not None else None, lo_format=self.lo_format,
                            post_scale=post[0] if post else None, post_shift=post[1] if post else None, post_relu=True,
                            range_flag=self.range_flag)
        nf = self.final.shape[-1]
        K.global_avgpool_nhwc(self.final, self.post_ss[0], self.post_ss[1], relu=True, out=self.total, ld_out=self.total.stride(0))
        theta = self.total[:, nf:]
        theta.copy_(self.mean_theta.expand(B, -1))                                                      # :245
        for _ in range(self.iterations):                                                                 # :246-248
            K.linear(self.total, self.fc[0][0], self.fc[0][1], relu=True, out=self.h1)
            K.linear(self.h1, self.fc[1][0], self.fc[1][1], relu=True, out=self.h2)
            K.linear(self.h2, self.fc[2][0], self.fc[2][1], relu=False, out=theta, accumulate=True)
        return theta.clone()


class HumanModelRecovery(StreamOwner, nn.Module):
    def __init__(self, smpl_pkl_path=None, feature_dim=2048, theta_dim=85, iterations=3, smpl_model=None):
        super(HumanModelRecovery, self).__init__()
        self.resnet = preActResNet50()
        self.smpl = SMPL(pkl_path=smpl_pkl_path, model=smpl_model)
        self.feature_dim = feature_dim
        self.theta_dim = theta_dim
        self.regressor = ThetaRegressor(feature_dim + theta_dim, theta_dim, iterations)
        self.iterations = iterations

    @torch.no_grad()
    def forward(self, inputs):
        """inputs [N,3,224,224] in [-1,1] -> theta [N,85] (networks/hmr.py:275-300)."""
        if self.training:
            raise LwbError("HumanModelRecovery runs in eval mode only (BatchNorm uses its running statistics)")
        if not inputs.is_cuda:
            raise LwbError("HumanModelRecovery runs on CUDA tensors only (no CPU fallback)")
        B = inputs.shape[0]
        split = split_mode(self)
        return stream_for(self, _HmrStream, (B, split), B, inputs.device, split, limit=2).run(inputs)

    def get_details(self, theta):
        cam = theta[:, 0:3].contiguous()
        pose = theta[:, 3:75].contiguous()
        shape = theta[:, 75:].contiguous()
        verts, j3d, rs = self.smpl(beta=shape, theta=pose, get_skin=True, cam=cam)
        return {'theta': theta, 'cam': cam, 'pose': pose, 'shape': shape, 'verts': verts,
                'j2d': self.smpl.j2d, 'j3d': j3d}
