"""Host-side mirror of models/swapper.py's ``Swapper`` (appearance transfer, inference only).

Person A (``src_info``) keeps pose, shape and the body parts that are NOT selected; the selected parts' appearance comes
from person B (``tsf_info``).  The generator runs its two-source form (``generator.swap``, networks/generator.py:245-275):
every Liquid Warping Block adds two warped feature sets -- B's features through ``T21`` (B's visible surface points looked
up through A's face-index map, selected parts only) and A's own features through ``T11`` (the identity grid on the parts A
keeps).  Reference surface mirrored here:

  Swapper(opt)                                                      models/swapper.py:22-60
  personalize(src_path, src_smpl=None, output_path='', visualizer=None) -> src_info   :99-165
  swap_smpl(src_cam, src_shape, tgt_smpl, preserve_scale=True)      :178-191
  swap_setup(src_path, tgt_path, src_smpl=None, tgt_smpl=None, output_dir='')          :194-196
  swap(src_info, tgt_info, target_part='body', visualizer=None) -> preds [1,3,H,W]     :199-239
  calculate_trans(src_left_mask, left_faces) -> T11, T21            :242-253
  warp / forward                                                    :255-270

``post_personalize`` (cycle fine-tuning) needs the backward pass and is out of scope.  The part table
(``mesh.create_mapping('par', opt.uv_mapping)``) and the per-part face lists come from the asset files like in the
reference; ``part_info=`` (dict part name -> {"face": [...]}) injects them instead (tests, no asset download).
"""
import torch

from . import mesh
from ._lib import LwbError
from .imitator import Imitator, _on_device


class Swapper(Imitator):

    PART_IDS = {
        'body': [1, 2, 3, 4, 5, 6, 7, 8, 9],
        'all': [0, 1, 2, 3, 4, 5, 6, 7, 8, 9]
    }

    def __init__(self, opt, part_info=None, **kw):
        super(Swapper, self).__init__(opt, **kw)
        self._name = 'Swapper'
        self.T = self.T12 = self.T21 = None
        self.grid = self.render.create_meshgrid(self._opt.image_size).to(self.device)
        if part_info is None:
            mapping = getattr(opt, 'uv_mapping', 'assets/pretrains/mapper.txt')
            part_fn = mesh.create_mapping('par', mapping, contain_bg=True, fill_back=False)
            self.part_faces_dict = mesh.get_part_face_ids(part_type='par', mapping_path=mapping, fill_back=False)
        else:
            names = sorted(part_info.keys())
            nf = self.render.nf
            import numpy as np
            part_fn = np.zeros((nf + 1, len(names) + 1), dtype=np.float32)
            for i, name in enumerate(names):
                part_fn[list(part_info[name]['face']), i] = 1.0
            part_fn[nf, -1] = 1.0                                      # background row (utils/mesh.py:404-410, 418-419)
            self.part_faces_dict = {name: list(part_info[name]['face']) for name in names}
        self.part_fn = torch.as_tensor(part_fn).float().to(self.device)
        self.part_faces = list(self.part_faces_dict.values())

    # ---- personalize: returns the info instead of storing it (models/swapper.py:99-165) --------
    @_on_device
    @torch.no_grad()
    def personalize(self, src_path, src_smpl=None, output_path='', visualizer=None, src_img=None, src_frame=None):
        return self._personalize(src_path, src_smpl, output_path, None, src_img, src_frame)

    def _extend_src_info(self, src_info):
        src_info['part'], _ = self.render.encode_fim(src_info['cam'], src_info['verts'], fim=src_info['fim'],
                                                     transpose=True, map_fn=self.part_fn)

    @torch.no_grad()
    def swap_smpl(self, src_cam, src_shape, tgt_smpl, preserve_scale=True):
        """models/swapper.py:178-191 (without its in-place edit of the caller's tgt_smpl)."""
        cam = tgt_smpl[:, 0:3].clone()
        pose = tgt_smpl[:, 3:75].contiguous()
        if preserve_scale:                                             # the reference's statement order: the ratio is 1
            cam[:, 0] = src_cam[:, 0]
            cam[:, 1:] = (src_cam[:, 0:1] / cam[:, 0:1]) * cam[:, 1:] + src_cam[:, 1:]
        return torch.cat([cam, pose, src_shape], dim=1)

    @_on_device
    @torch.no_grad()
    def swap_setup(self, src_path, tgt_path, src_smpl=None, tgt_smpl=None, output_dir='', src_img=None, tgt_img=None,
                   src_frame=None, tgt_frame=None):
        """``src_frame`` / ``tgt_frame`` (extension): uint8 [H,W,3] BGR frames in place of the files (Imitator.personalize)."""
        self.src_info = self.personalize(src_path, src_smpl, src_img=src_img, src_frame=src_frame)
        self.tsf_info = self.personalize(tgt_path, tgt_smpl, src_img=tgt_img, src_frame=tgt_frame)

    @_on_device
    @torch.no_grad()
    def swap(self, src_info, tgt_info, target_part='body', visualizer=None):
        if target_part not in self.PART_IDS:
            raise LwbError("target_part must be one of %r" % (sorted(self.PART_IDS),))
        selected_ids = self.PART_IDS[target_part]
        left_ids = [i for i in self.PART_IDS['all'] if i not in selected_ids]
        src_part_mask = (torch.sum(src_info['part'][:, selected_ids, ...], dim=1) != 0)
        if left_ids:
            src_left_mask = torch.sum(src_info['part'][:, left_ids, ...], dim=1).bool()
        else:
            src_left_mask = torch.zeros_like(src_part_mask)
        left_faces = sorted(set().union(*[set(self.part_faces[i]) for i in left_ids])) if left_ids else []

        T11, T21 = self.calculate_trans(src_left_mask, left_faces)
        tsf21 = self.generator.transform(tgt_info['img'], T21)
        tsf11 = self.generator.transform(src_info['img'], T11)
        part_f = src_part_mask[:, None, :, :].float()
        left_f = src_left_mask[:, None, :, :].float()
        tsf_img = tsf21 * part_f + tsf11 * left_f
        tsf_inputs = torch.cat([tsf_img, src_info['cond']], dim=1)
        preds, tsf_mask = self.forward(tsf_inputs, tgt_info['feats'], T21, src_info['feats'], T11, src_info['bg'])
        if getattr(self._opt, 'front_warp', False):
            preds = self.warp(preds, src_info['img'], src_info['fim'], tsf_mask)
        self.T11, self.T21 = T11, T21
        if visualizer is not None:
            visualizer.vis_named_img('src_img', src_info['img'])
            visualizer.vis_named_img('tgt_img', tgt_info['img'])
            visualizer.vis_named_img('preds', preds)
        return preds

    def calculate_trans(self, src_left_mask, left_faces):
        """T11: the identity grid where person A keeps its own parts, -2 elsewhere.  T21: for each pixel of A's image the
        point of B's image showing the same body-surface point, parts A keeps excluded (models/swapper.py:242-253)."""
        T11 = self.grid.clone()
        T11[~src_left_mask[0]] = -2
        T11 = T11[None]
        tsf_f2p = self.tsf_info['p2verts'].clone()
        if left_faces:
            tsf_f2p[0, torch.as_tensor(left_faces, dtype=torch.long, device=tsf_f2p.device)] = -2
        T21 = self.render.cal_bc_transform(tsf_f2p, self.src_info['fim'], self.src_info['wim'])
        T21.clamp_(-2, 2)
        return T11.contiguous(), T21.contiguous()

    def warp(self, preds, tsf, fim, fake_tsf_mask):
        front_mask = self.render.encode_front_fim(fim, transpose=True)
        return (1 - front_mask) * preds + tsf * front_mask * (1 - fake_tsf_mask)

    @_on_device
    @torch.no_grad()
    def forward(self, tsf_inputs, feats21, T21, feats11, T11, bg):
        src_encoder_outs21, src_resnet_outs21 = feats21
        src_encoder_outs11, src_resnet_outs11 = feats11
        tsf_color, tsf_mask, pred_imgs = self.generator.swap(tsf_inputs, src_encoder_outs21, src_encoder_outs11,
                                                             src_resnet_outs21, src_resnet_outs11, T21, T11, bg=bg)
        return pred_imgs, tsf_mask

    def inference(self, *a, **k):
        raise LwbError("Swapper has no inference(): use swap_setup() + swap() (models/swapper.py:194-239)")

    inference_by_smpls = inference
