"""Host-side mirror of models/imitator.py's ``Imitator`` (motion imitation, inference only).

Keeps the reference's public surface so ``run_imitator.py`` drives it unchanged:

  Imitator(opt)                                                         models/imitator.py:14-46
  personalize(src_path, src_smpl=None, output_path='', visualizer=None) :82-145
  inference(tgt_paths, tgt_smpls=None, cam_strategy='smooth', output_dir='', visualizer=None, verbose=True)
      -> list of float32 HxWx3 arrays in [-1, 1]                         :157-189
  inference_by_smpls(tgt_smpls, cam_strategy='smooth', output_dir='', visualizer=None)   :192-214
  swap_smpl / transfer_params_by_smpl / transfer_params / forward / warp_front           :216-342
  public state ``src_info`` / ``tsf_info`` (read by run_imitator.write_pair_info, run_imitator.py:33-45)

What changes is how the per-frame work executes: the reference loops over frames at batch 1,
launching >100 small kernels and syncing on ``.cpu()`` every frame (:166-179); here frames are
processed ``opt.batch_size`` at a time -- one fused correspondence pass (raster + cond + T + image
warp), one generator pass on the wgmma conv engine, one device->host copy per chunk -- and the
results are returned per frame, in order, with ``tsf_info`` describing the last frame.

``tgt_smpls=None`` (how run_imitator.py:239-241 calls it) sends the target images through the HMR encoder
(impersonator_b200.hmr, one batch per chunk).  ``opt.has_detector`` builds the Mask R-CNN person detector
(impersonator_b200.detectors, ks = ``opt.bg_ks``; weights from torch's hub cache) and ``personalize`` then takes the
background mask from its dilated body mask, as models/imitator.py:116-122 does.  Out of scope (SURVEY.md section 8):
``post_personalize`` (fine-tuning, needs backward).  Any object with ``__call__(img) -> theta`` and
``get_details(theta)`` can be injected as ``hmr`` (tests use a synthetic body model), and any object with
``inference(img) -> (bbox, body_mask)`` as ``detector``.
"""
import os

import numpy as np
import torch

from . import kernels as K
from ._lib import LwbError
from .generator import ImpersonatorGenerator, weights_epoch
from .nmr import SMPLRenderer


def _on_device(fn):
    """Run a method with the Imitator's device current: the kernels launch on the current device's stream."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *a, **k):
        if self.device.type == 'cuda' and self.device.index is not None and self.device.index != torch.cuda.current_device():
            with torch.cuda.device(self.device):
                return fn(self, *a, **k)
        return fn(self, *a, **k)
    return wrapped


def morph(src_bg_mask, ks, mode='erode'):
    """utils/util.py:73-89: box-filter erode / dilate of a {0,1} mask [N,1,H,W] (border counts as 1 / 0)."""
    pad = ks // 2
    x = torch.nn.functional.pad(src_bg_mask, [pad, pad, pad, pad], value=1.0 if mode == 'erode' else 0.0)
    pooled = torch.nn.functional.avg_pool2d(x, ks, stride=1) * (ks * ks)
    if mode == 'erode':
        return (pooled.round() == ks * ks).float()
    return (pooled.round() >= 1).float()


def _read_image(path, image_size):
    """cv_utils.read_cv2_img + transform_img (utils/cv_utils.py:10-47) -> RGB float32 CHW in [0,1], original."""
    import cv2
    img = cv2.imread(path, -1)
    if img is None:
        raise IOError("cannot read %s" % path)
    img = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
    x = cv2.resize(img, (image_size, image_size)).astype(np.float32) / 255.0
    return x.transpose((2, 0, 1)), img


def _save_image(img, path, image_size=None, normalize=False):
    """cv_utils.save_cv2_img (utils/cv_utils.py:23-36)."""
    import cv2
    img = cv2.cvtColor(img, cv2.COLOR_RGB2BGR)
    if image_size is not None:
        img = cv2.resize(img, (image_size, image_size))
    if normalize:
        img = ((img + 1) / 2.0 * 255).astype(np.uint8)
    cv2.imwrite(path, img)


class Imitator(object):
    """``Imitator(opt)`` builds everything from ``opt`` exactly like models/imitator.py:15-74 (+ models/models.py:64-76,
    159-179): generator through ``NetworksFactory`` + checkpoint, background net, HMR (+ SMPL), ``SMPLRenderer`` from the
    asset files.  The keyword arguments are an extension: any of them replaces the corresponding constructed object
    (tests and benchmarks inject synthetic networks / tables because every asset is an external download)."""

    def __init__(self, opt, generator=None, bgnet=None, hmr=None, render=None, device=None, detector=None):
        self._name = 'Imitator'
        self._opt = opt
        self._gpu_ids = getattr(opt, 'gpu_ids', '0')
        self._is_train = getattr(opt, 'is_train', False)
        self._save_dir = os.path.join(getattr(opt, 'checkpoints_dir', './outputs/checkpoints/'), getattr(opt, 'name', 'running'))
        self.device = torch.device(device if device is not None else 'cuda')
        self._G_cond_nc, self._D_cond_nc = self.cond_nc()
        self._create_networks(generator, bgnet, hmr, render, detector)
        self.src_info = None
        self.tsf_info = None
        self.first_cam = None

    @property
    def name(self):
        return self._name

    def cond_nc(self):
        """models/models.py:85-95."""
        map_name = getattr(self._opt, 'map_name', '')
        if map_name:
            from .mesh import get_map_fn_dim
            nc = get_map_fn_dim(map_name)
            return nc, nc
        nc = getattr(self._opt, 'cond_nc', 3)
        return nc, nc

    # ---- construction (models/imitator.py:25-74) -------------------------------------------------
    def _create_networks(self, generator=None, bgnet=None, hmr=None, render=None, detector=None):
        opt = self._opt
        self.generator = (generator if generator is not None else self._create_generator()).to(self.device).eval()
        if bgnet is not None:
            self.bgnet = bgnet.to(self.device).eval()
        elif getattr(opt, 'bg_model', 'ORIGINAL') != 'ORIGINAL':
            self.bgnet = self._create_bgnet().to(self.device).eval()
        else:
            self.bgnet = self.generator.bg_model
        if hmr is not None:
            self.hmr = hmr.to(self.device) if hasattr(hmr, 'to') else hmr
        else:
            self.hmr = self._create_hmr().to(self.device).eval()
        if render is None:
            render = SMPLRenderer(image_size=opt.image_size, tex_size=getattr(opt, 'tex_size', 3),
                                  has_front=getattr(opt, 'front_warp', False), fill_back=False)
        self.render = render.to(self.device)
        if detector is not None:
            self.detector = detector
        elif getattr(opt, 'has_detector', False):                       # models/imitator.py:43-46
            from .detectors import PersonMaskRCNNDetector
            self.detector = PersonMaskRCNNDetector(ks=getattr(opt, 'bg_ks', 13), threshold=0.5, to_gpu=False)
            self.detector.model = self.detector.model.to(self.device)
        else:
            self.detector = None

    def _create_bgnet(self):
        from .networks import NetworksFactory
        net = NetworksFactory.get_by_name('deepfillv2', c_dim=4)
        self._load_params(net, self._opt.bg_model, need_module=False)
        net.eval()
        return net

    def _create_generator(self):
        from .networks import NetworksFactory
        opt = self._opt
        net = NetworksFactory.get_by_name(getattr(opt, 'gen_name', 'impersonator'), bg_dim=4, src_dim=3 + self._G_cond_nc,
                                          tsf_dim=3 + self._G_cond_nc, repeat_num=getattr(opt, 'repeat_num', 6))
        load_path, load_epoch = getattr(opt, 'load_path', ''), getattr(opt, 'load_epoch', -1)
        if load_path:
            self._load_params(net, load_path)
        elif load_epoch > 0:
            self._load_network(net, 'G', load_epoch)
        else:
            raise ValueError('load_path {} is empty and load_epoch {} is 0'.format(load_path, load_epoch))
        net.eval()
        return net

    def _create_hmr(self):
        from .networks import HumanModelRecovery
        hmr = HumanModelRecovery(self._opt.smpl_model)
        saved_data = torch.load(self._opt.hmr_model, map_location='cpu')
        hmr.load_state_dict(saved_data)
        hmr.eval()
        return hmr

    def _load_network(self, network, network_label, epoch_label, need_module=False):
        """models/models.py:153-157."""
        load_path = os.path.join(self._save_dir, 'net_epoch_%s_id_%s.pth' % (epoch_label, network_label))
        self._load_params(network, load_path, need_module)

    @staticmethod
    def _load_params(network, load_path, need_module=False):
        """models/models.py:159-179."""
        assert os.path.exists(load_path), \
            'Weights file not found. Have you trained a model!? We are not providing one %s' % load_path
        save_data = torch.load(load_path, map_location='cpu')
        if need_module:
            network.load_state_dict(save_data)
        else:
            network.load_state_dict({(k[7:] if 'module' in k else k): v for k, v in save_data.items()})
        print('Loading net: %s' % load_path)

    @property
    def _ac(self):
        return K.default_align_corners()

    def _details(self, smpl):
        if self.hmr is None:
            raise LwbError("no body model: inject hmr= (HMR/SMPL need external files and are outside the hot path)")
        return self.hmr.get_details(smpl)

    # ---- personalize (models/imitator.py:82-145) ----------------------------------------------
    @_on_device
    @torch.no_grad()
    def personalize(self, src_path, src_smpl=None, output_path='', visualizer=None, src_img=None):
        self.src_info = self._personalize(src_path, src_smpl, output_path, visualizer, src_img)
        self.__dict__['_graphs'] = {}                    # captured chunk graphs hold the previous source's buffers

    def _original_bg(self, bg_inputs, img_bg):
        """--bg_model ORIGINAL: what the task keeps of the background net's output (models/imitator.py:130-131 keeps it
        as it is; models/viewer.py:129 pastes it under the visible background)."""
        return img_bg

    def _extend_src_info(self, src_info):
        """Task-specific additions to ``src_info`` (models/swapper.py:128-129 adds the part map)."""

    def _personalize(self, src_path, src_smpl=None, output_path='', visualizer=None, src_img=None):
        """The body shared by models/imitator.py:82-145, models/viewer.py:83-143 and models/swapper.py:99-165 -> src_info."""
        size = self._opt.image_size
        if src_img is None:
            img, ori_img = _read_image(src_path, size)
            img = torch.tensor(img * 2 - 1.0, dtype=torch.float32, device=self.device)[None, ...]
        else:
            img, ori_img = src_img.to(self.device).float(), None
        if src_smpl is None:
            if self.hmr is None or ori_img is None:
                raise LwbError("src_smpl required when no HMR network is injected")
            import cv2
            img_hmr = cv2.resize(ori_img, (224, 224)).astype(np.float32).transpose((2, 0, 1)) / 255.0 * 2 - 1.0
            src_smpl = self.hmr(torch.tensor(img_hmr, dtype=torch.float32, device=self.device)[None, ...])
        else:
            src_smpl = torch.as_tensor(src_smpl, dtype=torch.float32, device=self.device).reshape(1, -1)

        src_info = self._details(src_smpl)
        tabs = self.render.correspond(src_info['cam'], src_info['verts'], None, None, want_f2verts=True)
        src_info['fim'] = tabs['fim']
        src_info['wim'] = tabs['wim']
        src_info['cond'] = tabs['cond'].contiguous()
        src_info['f2verts'] = tabs['f2verts']
        p2verts = tabs['f2verts'][:, :, :, 0:2].clone()
        p2verts[:, :, :, 1] *= -1                                       # models/imitator.py:105-107
        src_info['p2verts'] = p2verts.contiguous()
        if getattr(self._opt, 'only_vis', False):
            src_info['p2verts'] = self.render.get_vis_f2pts(src_info['p2verts'], tabs['fim']).contiguous()
        self._extend_src_info(src_info)
        src_info['img'] = img
        src_info['image'] = ori_img

        if self.detector is not None:                                  # models/imitator.py:116-118
            _, body_mask = self.detector.inference(img[0])
            bg_mask = 1 - body_mask
        else:
            bg_mask = morph(src_info['cond'][:, -1:, :, :], ks=getattr(self._opt, 'bg_ks', 13), mode='erode')
            body_mask = 1 - bg_mask
        if self.bgnet is self.generator.bg_model:
            bg_inputs = torch.cat([img * bg_mask, bg_mask], dim=1)
            src_info['bg'] = self._original_bg(bg_inputs, self.bgnet(bg_inputs))
        else:
            src_info['bg'] = self.bgnet(img, masks=body_mask, only_x=True)
        ft_mask = 1 - morph(src_info['cond'][:, -1:, :, :], ks=getattr(self._opt, 'ft_ks', 3), mode='erode')
        src_inputs = torch.cat([img * ft_mask, src_info['cond']], dim=1)
        src_info['src_inputs'] = src_inputs
        src_info['feats'] = self.generator.encode_src(src_inputs)
        if visualizer is not None:
            visualizer.vis_named_img('src', img)
            visualizer.vis_named_img('bg', src_info['bg'])
        if output_path and ori_img is not None:
            _save_image(ori_img, output_path, image_size=size)
        return src_info

    # ---- per-frame geometry (models/imitator.py:216-268) --------------------------------------
    def swap_smpl(self, src_cam, src_shape, tgt_smpl, cam_strategy='smooth'):
        tgt_cam = tgt_smpl[:, 0:3].contiguous()
        pose = tgt_smpl[:, 3:75].contiguous()
        if cam_strategy == 'smooth':
            cam = src_cam.expand(tgt_smpl.shape[0], -1).clone()
            cam[:, 1:] += tgt_cam[:, 1:] - self.first_cam[:, 1:]
        elif cam_strategy == 'source':
            cam = src_cam.expand(tgt_smpl.shape[0], -1)
        else:
            cam = tgt_cam
        return torch.cat([cam, pose, src_shape.expand(tgt_smpl.shape[0], -1)], dim=1)

    @_on_device
    @torch.no_grad()
    def transfer_params_by_smpl(self, tgt_smpl, cam_strategy='smooth', t=0):
        """tgt_smpl [85] or [B,85]: one frame (reference) or a chunk of frames (batched fast path)."""
        src_info = self.src_info
        tgt_smpl = torch.as_tensor(tgt_smpl, dtype=torch.float32, device=self.device)
        if tgt_smpl.dim() == 1:
            tgt_smpl = tgt_smpl[None, ...]
        if t == 0 and cam_strategy == 'smooth':
            self._set_first_cam(tgt_smpl[0:1, 0:3])
        tsf_smpl = self.swap_smpl(src_info['cam'], src_info['shape'], tgt_smpl, cam_strategy=cam_strategy)
        tsf_info = self._details(tsf_smpl)
        out = self.render.correspond(tsf_info['cam'], tsf_info['verts'], src_info['p2verts'], src_info['img'],
                                     align_corners=self._ac)
        tsf_info['fim'] = out['fim']
        tsf_info['wim'] = out['wim']
        tsf_info['cond'] = out['cond']
        tsf_info['tsf_img'] = out['tsf_img']
        tsf_info['T'] = out['T']
        self.tsf_info = tsf_info
        return out['tsf_inputs']

    def _set_first_cam(self, cam):
        """models/imitator.py:243-244, into a persistent buffer (a captured CUDA graph reads it at a fixed address)."""
        buf = getattr(self, '_first_cam_buf', None)
        if buf is None or buf.device != cam.device:
            buf = self._first_cam_buf = torch.empty((1, 3), dtype=torch.float32, device=cam.device)
        buf.copy_(cam)
        self.first_cam = buf

    def _chunk_pure(self, smpl, cam_strategy='smooth', hwc=True, u8=False):
        """Everything one chunk of frames needs on the device, as a pure function of the SMPL vectors [B,85] (no host sync,
        persistent or pool-allocated buffers only: capturable as a CUDA graph): camera swap, SMPL LBS, raster +
        correspondence, generator + composite, output-path layouts, range-flag snapshot."""
        src_info = self.src_info
        tsf_smpl = self.swap_smpl(src_info['cam'], src_info['shape'], smpl, cam_strategy=cam_strategy)
        tsf_info = self._details(tsf_smpl)
        out = self.render.correspond(tsf_info['cam'], tsf_info['verts'], src_info['p2verts'], src_info['img'],
                                     align_corners=self._ac)
        tsf_info['fim'], tsf_info['wim'], tsf_info['cond'] = out['fim'], out['wim'], out['cond']
        tsf_info['tsf_img'], tsf_info['T'] = out['tsf_img'], out['T']
        self.tsf_info = tsf_info
        preds = self._forward_chunk(out['tsf_inputs'], out['T'], host_layout=dict(hwc=hwc, u8=u8))
        flag = self.generator.tsf_model.range_flag_tensor()            # operand-range bits of this chunk's pass
        flag = flag.clone() if flag is not None else None              # snapshot: the next pass zeroes the live flag
        return dict(tsf_info=tsf_info, preds=preds, hwc=self._out_hwc, u8=self._out_u8, flag=flag)

    def _chunk_step(self, smpl, cam_strategy, hwc, u8):
        """``_chunk_pure`` eagerly, or -- LWB_GRAPH, full chunks -- replayed from a CUDA graph captured once per
        (batch, camera strategy, layouts, source).  Graph outputs are static buffers: the frames / flag are staged into fresh
        tensors here so that the D2H of this chunk may overlap the next replay."""
        from .graph import CapturedStep, graphs_enabled
        B = smpl.shape[0]
        bs = max(1, int(getattr(self._opt, 'batch_size', 1)))
        if not graphs_enabled() or B != bs or getattr(self._opt, 'front_warp', False):
            return self._chunk_pure(smpl, cam_strategy, hwc, u8)
        graphs = self.__dict__.setdefault('_graphs', {})
        key = (B, int(smpl.shape[1]), cam_strategy, bool(hwc), bool(u8), id(self.src_info), os.environ.get("LWB_PRECISION"),
               os.environ.get("LWB_STREAMS"), self._ac, getattr(self.generator, '_lwb_precision', None), weights_epoch())
        step = graphs.get(key)
        if step is None:
            if len(graphs) >= 4:
                graphs.pop(next(iter(graphs)))
            step = graphs[key] = CapturedStep(lambda smpl: self._chunk_pure(smpl, cam_strategy, hwc, u8), dict(smpl=smpl))
        res = step(smpl=smpl)
        if not step.captured:
            return res
        self.tsf_info = res['tsf_info']
        stage = lambda t: t.clone() if t is not None else None
        return dict(tsf_info=res['tsf_info'], preds=res['preds'], hwc=stage(res['hwc']), u8=stage(res['u8']), flag=stage(res['flag']))

    @torch.no_grad()
    def transfer_params(self, tgt_path, tgt_smpl=None, cam_strategy='smooth', t=0):
        ori_img = None
        if tgt_path:
            _, ori_img = _read_image(tgt_path, self._opt.image_size)
        if tgt_smpl is None:
            if self.hmr is None or ori_img is None:
                raise LwbError("tgt_smpl required when no HMR network is injected")
            import cv2
            img_hmr = cv2.resize(ori_img, (224, 224)).astype(np.float32).transpose((2, 0, 1)) / 255.0 * 2 - 1.0
            tgt_smpl = self.hmr(torch.tensor(img_hmr, dtype=torch.float32, device=self.device)[None, ...])
        tsf_inputs = self.transfer_params_by_smpl(tgt_smpl=tgt_smpl, cam_strategy=cam_strategy, t=t)
        self.tsf_info['image'] = ori_img
        return tsf_inputs

    # ---- generator + composite (models/imitator.py:326-342) -----------------------------------
    @_on_device
    @torch.no_grad()
    def forward(self, tsf_inputs, T):
        """models/imitator.py:326-336 -> preds [B,3,H,W]."""
        return self._forward_chunk(tsf_inputs, T)

    @_on_device
    @torch.no_grad()
    def _forward_chunk(self, tsf_inputs, T, host_layout=None):
        """-> preds [B,3,H,W].  ``host_layout`` = dict(hwc=bool, u8=bool) additionally fills
        ``self._out_hwc`` / ``self._out_u8`` ([B,H,W,3] float32 / uint8 BGR, the output path of
        models/imitator.py:178-187) -- from the head kernel itself unless warp_front rewrites the frames."""
        enc, res = self.src_info['feats']
        front = getattr(self._opt, 'front_warp', False)
        hwc = u8 = None
        if host_layout:
            B, _, H, W = tsf_inputs.shape
            hwc = torch.empty((B, H, W, 3), dtype=torch.float32, device=self.device) if host_layout.get('hwc') else None
            u8 = torch.empty((B, H, W, 3), dtype=torch.uint8, device=self.device) if host_layout.get('u8') else None
        if front or not host_layout:
            color, mask, pred = self.generator.inference(enc, res, tsf_inputs, T, bg=self.src_info['bg'])
            if front:
                pred = Imitator.warp_front(self, pred, mask)     # subclasses (Viewer) redefine warp_front's signature
            if host_layout:
                from . import kernels as K
                hwc, u8 = K.frames_out(pred.contiguous(), want_hwc=hwc is not None, want_u8=u8 is not None)
        else:
            color, mask, pred = self.generator.inference(enc, res, tsf_inputs, T, bg=self.src_info['bg'],
                                                         pred_hwc=hwc, pred_u8=u8)
        self._out_hwc, self._out_u8 = hwc, u8
        return pred

    def warp_front(self, preds, mask):
        front_mask = self.render.encode_front_fim(self.tsf_info['fim'], transpose=True, front_fn=True)
        return (1 - front_mask) * preds + self.tsf_info['tsf_img'] * front_mask * (1 - mask)

    # ---- the hot loop (models/imitator.py:157-214), chunked -----------------------------------
    def _chunks(self, n):
        bs = max(1, int(getattr(self._opt, 'batch_size', 1)))
        return [(i, min(n, i + bs)) for i in range(0, n, bs)]

    @_on_device
    @torch.no_grad()
    def inference(self, tgt_paths, tgt_smpls=None, cam_strategy='smooth', output_dir='', visualizer=None, verbose=True,
                  as_uint8=False, score_against=None, lpips=None):
        """models/imitator.py:157-189.  Returns per-frame float32 HxWx3 arrays in [-1,1] like the reference; with
        ``as_uint8=True`` (extra) returns the BGR uint8 images the reference writes to disk instead (4x less D2H).
        With ``output_dir`` the uint8 images come from the GPU and go straight to cv2.imwrite.

        ``score_against`` (extra): ground-truth frames [N,3,H,W] in [-1,1] (numpy or tensor, N = len(tgt_paths)).  Each
        chunk's frames are scored while still on the device (impersonator_b200.metrics.score_frames: SSIM and PSNR, and
        LPIPS when an ``lpips`` = metrics.LPIPS is given), and the call returns (outputs, scores) with scores a dict of
        per-frame float64 numpy arrays."""
        length = len(tgt_paths)
        if score_against is not None:
            from . import metrics as _metrics
            if len(score_against) != length:
                raise LwbError("score_against holds %d frames for %d targets" % (len(score_against), length))
            scores = []
        outputs = []
        last_image = [None]
        originals = {}                                           # frame index -> original RGB image (for the gt_ files)

        def chunk_smpls(a, b):
            """SMPL vectors of frames a..b-1: given, or estimated from the target images by HMR -- one encoder batch per
            chunk instead of one launch sequence per frame (models/imitator.py:271-275)."""
            if tgt_smpls is not None:
                return torch.as_tensor(np.stack([np.asarray(s, dtype=np.float32).reshape(-1) for s in tgt_smpls[a:b]]))
            if self.hmr is None or not callable(self.hmr):
                raise LwbError("tgt_smpls required when no HMR network is available")
            import cv2
            batch = []
            for k, path in enumerate(tgt_paths[a:b]):
                _, ori = _read_image(path, self._opt.image_size)
                batch.append(cv2.resize(ori, (224, 224)).astype(np.float32).transpose((2, 0, 1)) / 255.0 * 2 - 1.0)
                last_image[0] = ori
                if output_dir:
                    originals[a + k] = ori
            return self.hmr(torch.from_numpy(np.stack(batch)).to(self.device))
        # Chunks are pipelined: the D2H of chunk i runs on a copy stream while chunk i+1 computes; the host only
        # waits for a chunk's copy when it has already queued the next chunk (and once at the end).
        main = torch.cuda.current_stream(self.device)
        if getattr(self, '_copy_stream', None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        pending = []
        range_bits = [0]

        def drain(keep):
            while len(pending) > keep:
                a0, b0, h_f, h_u8, h_flag, done = pending.pop(0)
                done.synchronize()
                if h_flag is not None:
                    range_bits[0] |= int(h_flag[0])
                host = h_u8 if as_uint8 else h_f
                for j in range(b0 - a0):
                    outputs.append(host[j])
                    if output_dir:
                        self._maybe_save(h_u8[j], tgt_paths[a0 + j], output_dir, a0 + j, is_bgr_u8=True,
                                         original=originals.pop(a0 + j, None))

        for (a, b) in self._chunks(length):
            smpls = torch.as_tensor(chunk_smpls(a, b), dtype=torch.float32).to(self.device, non_blocking=True)
            if smpls.dim() == 1:
                smpls = smpls[None, ...]
            if a == 0 and cam_strategy == 'smooth':
                self._set_first_cam(smpls[0:1, 0:3])
            want_u8 = bool(as_uint8 or output_dir)
            res = self._chunk_step(smpls, cam_strategy, not as_uint8, want_u8)
            out_hwc, out_u8, flag = res['hwc'], res['u8'], res['flag']
            if score_against is not None:
                gt = _metrics._frames(score_against[a:b], self.device)
                scores.append(_metrics.score_frames(res['preds'], gt, from01=False, lpips=lpips))
            if visualizer is not None:
                visualizer.vis_named_img('pred_' + cam_strategy, res['preds'])
            ready = torch.cuda.Event()
            ready.record(main)
            with torch.cuda.stream(self._copy_stream):
                self._copy_stream.wait_event(ready)
                h_f = self._to_host(out_hwc, sync=False) if not as_uint8 else None
                h_u8 = self._to_host(out_u8, sync=False) if want_u8 else None
                h_flag = self._to_host(flag, sync=False) if flag is not None else None
                for t in (out_hwc, out_u8, flag):
                    if t is not None:
                        t.record_stream(self._copy_stream)
                done = torch.cuda.Event()
                done.record(self._copy_stream)
            pending.append((a, b, h_f, h_u8, h_flag, done))
            drain(keep=1)
        drain(keep=0)

        def result():
            if score_against is None:
                return outputs
            keys = scores[0].keys() if scores else ("ssim", "psnr")
            return outputs, {k: torch.cat([s[k].double() for s in scores]).cpu().numpy() if scores else np.zeros(0)
                             for k in keys}
        self._last_frame_info()
        if last_image[0] is None and length and tgt_paths[-1] and self.tsf_info:
            # driven by given SMPL vectors AND frame files (evaluate.py:62): transfer_params still reads every frame file
            # (models/imitator.py:270) and leaves the last one in tsf_info['image']; only that one is read here
            _, last_image[0] = _read_image(tgt_paths[-1], self._opt.image_size)
        if last_image[0] is not None:
            self.tsf_info['image'] = last_image[0]
        if range_bits[0] and not getattr(self, '_range_retry', False):
            # Never silently: activations left the range in which the default fp16f8 operand split keeps its precision
            # (bit 0: |x| >= 1024, the e4m3 correction terms clip; bit 2: output-head pre-activations of +-8 and more, where
            # its ~1e-4 relative precision may exceed 1e-3 on pixels).  Pin the generator to fp16x3 (fp16 corrections, range
            # 6e4) and redo the call -- LWB_AUTO_PRECISION=0 only warns; beyond the fp16 range (bit 1) nothing in this
            # engine can represent the activations.
            import warnings
            if range_bits[0] & 2:
                raise LwbError("generator activations exceed the fp16 range (|x| >= 6e4 or non-finite): the conv engine's "
                               "fp16 operands cannot represent them")
            what = ("activations beyond the fp16f8 correction range (|x| >= 1024)" if range_bits[0] & 1 else
                    "output-head pre-activations beyond +-8 (fp16f8's ~1e-4 relative precision may exceed 1e-3 on pixels)")
            if os.environ.get("LWB_AUTO_PRECISION", "1") == "0" or getattr(self.generator, '_lwb_precision', None) == "fp16x3" \
                    or os.environ.get("LWB_PRECISION", "fp16f8") != "fp16f8":
                warnings.warn("lwb_b200: %s (precision mode kept)" % what)
                return result()
            warnings.warn("lwb_b200: %s; switching this generator to LWB_PRECISION=fp16x3 and recomputing the sequence" % what)
            self.generator.set_precision("fp16x3")
            self._range_retry = True
            try:
                enc_in = self.src_info.get('src_inputs')
                if enc_in is not None:
                    self.src_info['feats'] = self.generator.encode_src(enc_in)
                return self.inference(tgt_paths, tgt_smpls, cam_strategy, output_dir, visualizer, verbose, as_uint8,
                                      score_against, lpips)
            finally:
                self._range_retry = False
        return result()

    @torch.no_grad()
    def inference_by_smpls(self, tgt_smpls, cam_strategy='smooth', output_dir='', visualizer=None, as_uint8=False):
        return self.inference([''] * len(tgt_smpls), tgt_smpls, cam_strategy, output_dir, visualizer, verbose=False,
                              as_uint8=as_uint8)

    @staticmethod
    def _to_host(t, sync=True):
        """Device -> pinned host (torch's caching host allocator), one async copy on the current stream (+ one sync)."""
        h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        h.copy_(t, non_blocking=True)
        if sync:
            torch.cuda.current_stream().synchronize()
        return h.numpy()

    def _last_frame_info(self):
        """tsf_info must describe the LAST frame (run_imitator.py:33-45 reads fim/T/tsf_img/cam/verts/wim)."""
        if not self.tsf_info:                              # empty sequence: nothing was rendered
            return
        info = dict(self.tsf_info)
        for k, v in list(info.items()):
            if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] >= 1:
                info[k] = v[-1:].clone()                 # own storage: the chunk buffers may belong to a replayed graph
        self.tsf_info = info

    def _maybe_save(self, pred, tgt_path, output_dir, t, is_bgr_u8=False, original=None):
        """pred_<file> (+ gt_<file> = the driving frame resized, models/imitator.py:182-187); inference_by_smpls names
        its frames pred_%.8d.jpg (:212)."""
        if not output_dir:
            return
        name = os.path.split(tgt_path)[-1] if tgt_path else 'pred_%.8d.jpg' % t
        path = os.path.join(output_dir, 'pred_' + name if tgt_path else name)
        if tgt_path:
            if original is None:
                _, original = _read_image(tgt_path, self._opt.image_size)
            _save_image(original, os.path.join(output_dir, 'gt_' + name), image_size=self._opt.image_size)
        if is_bgr_u8:
            import cv2
            cv2.imwrite(path, pred)                      # already what save_cv2_img(normalize=True) would write
        else:
            _save_image(pred, path, normalize=True)

    def post_personalize(self, *a, **k):
        raise LwbError("post_personalize (fine-tuning) needs the backward pass: outside the inference hot path")


class SyntheticBodyModel(object):
    """Stand-in for ``HumanModelRecovery.get_details`` (networks/hmr.py:302-330) when SMPL's model files
    are absent: theta[0:3] = cam, theta[3:6] = (ry, rx, k) pose parameters of the synthetic UV-sphere
    body (impersonator_b200.synthetic), theta[75:85] = shape (ignored)."""

    def __init__(self, base_verts):
        self.base = base_verts
        self._on = {}

    def get_details(self, theta):
        dev = theta.device
        if dev not in self._on:                          # one upload per device (a per-call H2D copy cannot be graph-captured)
            self._on[dev] = self.base.to(dev)
        base = self._on[dev]
        cam = theta[:, 0:3].contiguous()
        ry, rx = theta[:, 3], theta[:, 4]
        cy, sy, cx, sx = torch.cos(ry), torch.sin(ry), torch.cos(rx), torch.sin(rx)
        zeros, ones = torch.zeros_like(cy), torch.ones_like(cy)
        Ry = torch.stack([cy, zeros, sy, zeros, ones, zeros, -sy, zeros, cy], dim=1).view(-1, 3, 3)
        Rx = torch.stack([ones, zeros, zeros, zeros, cx, -sx, zeros, sx, cx], dim=1).view(-1, 3, 3)
        verts = base[None] @ Ry.transpose(1, 2) @ Rx.transpose(1, 2)
        return {'theta': theta, 'cam': cam, 'pose': theta[:, 3:75].contiguous(), 'shape': theta[:, 75:].contiguous(),
                'verts': verts.contiguous(), 'j2d': None, 'j3d': None}
