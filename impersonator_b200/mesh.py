"""Face lookup tables of ``SMPLRenderer`` built from the asset files, as ``utils/mesh.py`` does (pure numpy, load time).

  load_obj(path)                       utils/mesh.py:28-79    (``v`` / ``vn`` / ``vt`` / ``f a/b/c`` records of mapper.txt)
  get_f2vts(path, fill_back)           :175-197               per-face uv triangle, v flipped (1 - v), z = 0
  compute_barycenter(f2vts)            :159-172
  create_mapping(map_name, ...)        :368-421               'uv_seg' (what the generator is conditioned on), 'uv', 'seg',
                                                              'front', 'head', 'back', 'par', 'ids', 'binary'
  get_map_fn_dim(map_name)             :446-473
Only what the hot path's constructor needs is here (``SMPLRenderer.__init__``, utils/nmr.py:104-178); texture samplers
(create_uvsampler) belong to the textured-rendering path, which is out of scope.
"""
import json
import os

import numpy as np


def load_obj(obj_file):
    verts, faces, vts, vns, faces_vts, faces_vns = [], [], [], [], [], []
    with open(obj_file, 'r') as fp:
        for line in fp:
            parts = line.rstrip().split()
            if not parts:
                continue
            tag = parts[0]
            if tag == 'v':
                verts.append([float(t) for t in parts[1:4]])
            elif tag == 'vn':
                vns.append([float(t) for t in parts[1:4]])
            elif tag == 'vt':
                vts.append([float(t) for t in parts[1:3]])
            elif tag == 'f':
                idx = [p.split('/') for p in parts[1:4]]
                faces.append([int(p[0]) - 1 for p in idx])
                faces_vts.append([int(p[1]) - 1 for p in idx])
                faces_vns.append([int(p[2]) - 1 for p in idx])
            else:
                raise ValueError(tag)                      # the reference rejects any other record, utils/mesh.py:66
    return {'vertices': np.array(verts, dtype=np.float32), 'faces': np.array(faces, dtype=np.int32),
            'vts': np.array(vts, dtype=np.float32), 'vns': np.array(vns, dtype=np.float32),
            'faces_vts': np.array(faces_vts, dtype=np.int32), 'faces_vns': np.array(faces_vns, dtype=np.int32)}


def get_f2vts(uv_mapping_path, fill_back=False):
    """-> F x 3 x 3: the uv triangle of every face (v axis flipped, z = 0)."""
    obj = load_obj(uv_mapping_path)
    vts = obj['vts'].copy()
    vts[:, 1] = 1 - vts[:, 1]
    vts = np.concatenate([vts, np.zeros((vts.shape[0], 1), dtype=np.float32)], axis=-1)
    faces = obj['faces_vts']
    if fill_back:
        faces = np.concatenate((faces, faces[:, ::-1]), axis=0)
    return vts[faces]


def compute_barycenter(f2vts):
    v2 = f2vts[:, 2]
    return v2 + 0.5 * (f2vts[:, 0] - v2) + 0.5 * (f2vts[:, 1] - v2)


def _face_set(path):
    with open(path, 'r') as fp:
        return list(json.load(fp)['face'])


def _mask(nf, faces, fill_back):
    table = np.zeros((nf, 1), dtype=np.float32)
    faces = list(faces)
    if fill_back:
        faces = faces + [f + nf // 2 for f in faces]
    table[faces] = 1.0
    return table, np.zeros((1, 1), dtype=np.float32)


def _sibling(mapping_path, name, default):
    """The reference hard-codes 'assets/pretrains/<name>' (utils/mesh.py:369-371); the same file next to the mapper wins
    when the mapper lives elsewhere."""
    cand = os.path.join(os.path.dirname(mapping_path), name)
    return cand if os.path.exists(cand) else default


def create_mapping(map_name, mapping_path='assets/pretrains/mapper.txt', part_info=None, front_info=None, head_info=None,
                   contain_bg=True, fill_back=False):
    part_info = part_info or _sibling(mapping_path, 'smpl_part_info.json', 'assets/pretrains/smpl_part_info.json')
    front_info = front_info or _sibling(mapping_path, 'front_facial.json', 'assets/pretrains/front_facial.json')
    head_info = head_info or _sibling(mapping_path, 'head.json', 'assets/pretrains/head.json')
    f2vts = get_f2vts(mapping_path, fill_back=fill_back)
    nf = f2vts.shape[0]
    if map_name == 'uv':
        map_fn, bg = compute_barycenter(f2vts)[:, 0:2], np.array([[-1, -1]], dtype=np.float32)
    elif map_name == 'seg':
        map_fn, bg = np.ones((nf, 1), dtype=np.float32), np.array([[0]], dtype=np.float32)
    elif map_name == 'uv_seg':
        map_fn, bg = compute_barycenter(f2vts), np.array([[0, 0, 1]], dtype=np.float32)
    elif map_name == 'par':
        with open(part_info, 'r') as fp:
            parts = json.load(fp)
        names = sorted(parts.keys())
        map_fn = np.zeros((nf, len(names) + 1), dtype=np.float32)
        seen = set()
        for i, name in enumerate(names):
            faces = list(parts[name]['face'])
            map_fn[faces, i] = 1.0
            seen |= set(faces)
        assert len(seen) == nf, 'nf_counter = {}, nf = {}'.format(len(seen), nf)
        bg = np.zeros((1, len(names) + 1), dtype=np.float32)
        bg[0, -1] = 1
    elif map_name == 'front':
        map_fn, bg = _mask(nf, _face_set(front_info), fill_back)
    elif map_name == 'head':
        map_fn, bg = _mask(nf, _face_set(head_info), fill_back)
    elif map_name == 'back':
        map_fn, bg = _mask(nf, set(_face_set(head_info)) - set(_face_set(front_info)), fill_back)
    elif map_name == 'ids':
        # one column (the reference's 1-D arange cannot be stacked on its [1, 1] background row); np.arange with a float
        # step may return nf + 1 values
        map_fn, bg = np.arange(0, 1, 1 / nf, dtype=np.float32)[:nf, None], np.array([[-1]], dtype=np.float32)
    elif map_name == 'binary':
        # the face index in at least get_map_fn_dim('binary') = 15 bits, the width the generator is built for (the
        # reference codes it in len(binary_repr(nf)) bits: 14 for the 13776 SMPL faces, one column short of its generator)
        width = max(len(np.binary_repr(nf)), get_map_fn_dim('binary'))
        map_fn = np.stack([np.array(list(map(int, np.binary_repr(i, width=width)))) for i in range(nf)], axis=0)
        bg = np.zeros((1, width), dtype=np.float32) - 1.0
    else:
        raise ValueError('map name error {}'.format(map_name))
    if contain_bg:
        map_fn = np.concatenate([map_fn, bg], axis=0)
    return map_fn


def get_part_face_ids(part_type, mapping_path='assets/pretrains/mapper.txt', part_info=None, front_info=None, head_info=None,
                      fill_back=False):
    """utils/mesh.py:424-443 (+ :247-268, :327-365): the face ids of a part selection.  'par' -> ordered dict
    part name -> face list (the parts must cover every face once); 'head_front' / 'head_back' -> face list."""
    part_info = part_info or _sibling(mapping_path, 'smpl_part_info.json', 'assets/pretrains/smpl_part_info.json')
    front_info = front_info or _sibling(mapping_path, 'front_face_1.json', 'assets/pretrains/front_face_1.json')
    head_info = head_info or _sibling(mapping_path, 'head.json', 'assets/pretrains/head.json')
    nf = get_f2vts(mapping_path, fill_back=fill_back).shape[0]
    half = nf // 2

    def both_sides(faces):
        faces = list(faces)
        return faces + [f + half for f in faces] if fill_back else faces

    if part_type == 'par':
        with open(part_info, 'r') as fp:
            parts = json.load(fp)
        ordered, seen = {}, set()
        for name in sorted(parts.keys()):
            ordered[name] = both_sides(parts[name]['face'])
            seen |= set(ordered[name])
        assert len(seen) == nf, 'nf_counter = {}, nf = {}'.format(len(seen), nf)
        return ordered
    if part_type == 'head_front':
        return both_sides(_face_set(front_info))
    if part_type == 'head_back':
        return both_sides(set(_face_set(head_info)) - set(_face_set(front_info)))
    if part_type == 'head':
        raise NotImplementedError
    raise ValueError('map name error {}'.format(part_type))


def get_map_fn_dim(map_name):
    dims = {'seg': 1, 'uv': 2, 'uv_seg': 3, 'par': 11, 'ids': 1, 'binary': 15}
    if map_name not in dims:
        raise ValueError('map name error {}'.format(map_name))
    return dims[map_name]
