"""Register two point clouds with a 3DMatch snapshot, the experiment's ``demo.py``.

    python -m geotransformer_b200.demo --src-file SRC.npy --ref-file REF.npy [--gt-file GT.npy] --weights FILE \\
        [--voxel-size V] [--output DIR [--normals]]

Ones as features, the 3DMatch config's fixed neighbour limits [38, 36, 36, 38] and ``state_dict['model']`` of the snapshot, as the
reference.  ``--voxel-size`` first downsamples both clouds on the device with Open3D's voxel downsampling
(``utils.open3d.voxel_downsample``), for clouds that are not already at the training voxel size.  With ``--gt-file`` the reference's
``RRE(deg): ..., RTE(m): ...`` line is printed.  Instead of Open3D windows, ``--output`` writes ``estimated_transform.npy`` and
``registration.ply``: an ASCII PLY of the ref points in ``custom_yellow`` and the src points aligned by the estimate in
``custom_blue``.  With ``--normals`` the PLY also holds ``nx ny nz``, so it can be viewed shaded as the reference shows it: the
ref normals are ``utils.open3d.estimate_normals(ref)``, the src normals are estimated on the unaligned src and rotated by the
estimate's R, as Open3D's ``PointCloud.transform`` does in the reference demo.  3DMatch only, as the reference's demo: KITTI's neighbour limits are calibrated, not fixed.
"""
import argparse
import os

import numpy as np
import torch

from .config import make_cfg
from .utils.data import registration_collate_fn_stack_mode

CUSTOM_YELLOW = (255, 204, 102)   # reference utils/open3d.py get_color, times 255
CUSTOM_BLUE = (102, 153, 255)


def load_data(src_file, ref_file, gt_file=None, voxel_size=None):
    """the reference demo's data dict; with ``voxel_size`` both clouds are voxel-downsampled on the device first"""
    src_points = np.load(src_file)
    ref_points = np.load(ref_file)
    if voxel_size is not None:
        from .utils.open3d import voxel_downsample
        src_points = voxel_downsample(src_points, voxel_size)
        ref_points = voxel_downsample(ref_points, voxel_size)
    data_dict = {
        'ref_points': ref_points.astype(np.float32),
        'src_points': src_points.astype(np.float32),
        'ref_feats': np.ones_like(ref_points[:, :1]).astype(np.float32),
        'src_feats': np.ones_like(src_points[:, :1]).astype(np.float32),
    }
    if gt_file is not None:
        data_dict['transform'] = np.load(gt_file).astype(np.float32)
    return data_dict


def write_ply(path, ref_points, src_points, ref_normals=None, src_normals=None):
    """ASCII PLY: ref in custom_yellow, then src in custom_blue; with normals (both or neither) also nx ny nz per vertex"""
    rows = [(p, CUSTOM_YELLOW) for p in ref_points] + [(p, CUSTOM_BLUE) for p in src_points]
    normals = None if ref_normals is None else list(ref_normals) + list(src_normals)
    with open(path, 'w') as f:
        f.write('ply\nformat ascii 1.0\n')
        f.write(f'element vertex {len(rows)}\n')
        f.write('property float x\nproperty float y\nproperty float z\n')
        if normals is not None:
            f.write('property double nx\nproperty double ny\nproperty double nz\n')
        f.write('property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n')
        for r, (p, c) in enumerate(rows):
            nrm = '' if normals is None else f'{float(normals[r][0]):.17g} {float(normals[r][1]):.17g} {float(normals[r][2]):.17g} '
            f.write(f'{float(p[0]):.9g} {float(p[1]):.9g} {float(p[2]):.9g} {nrm}{c[0]} {c[1]} {c[2]}\n')


def registration_normals(ref_points, src_points, estimated_transform):
    """the shaded view's normals: ref's from estimate_normals, src's estimated on the unaligned src and rotated by the estimate's R
    in double (Open3D's TransformNormals); both (N, 3) float64 numpy"""
    from .utils.open3d import estimate_normals
    ref_normals = estimate_normals(np.asarray(ref_points))
    src_normals = estimate_normals(np.asarray(src_points))
    R = np.asarray(estimated_transform)[:3, :3].astype(np.float64)
    return ref_normals, src_normals @ R.T


def run(src_file, ref_file, weights, gt_file=None, voxel_size=None, output=None, normals=False):
    """the demo; returns (estimated transform (4, 4) float32 numpy, (rre, rte) or None)"""
    from .model import create_model
    from .utils.registration import compute_registration_error
    cfg = make_cfg('3dmatch')
    data_dict = load_data(src_file, ref_file, gt_file, voxel_size)
    neighbor_limits = [38, 36, 36, 38]  # default setting in 3DMatch
    data_dict = registration_collate_fn_stack_mode([data_dict], cfg.backbone.num_stages, cfg.backbone.init_voxel_size,
                                                   cfg.backbone.init_radius, neighbor_limits)
    model = create_model(cfg).cuda()
    state_dict = torch.load(weights, map_location='cpu')
    model.load_state_dict(state_dict['model'])
    model.eval()
    output_dict = model(data_dict)
    estimated_transform = output_dict['estimated_transform'].cpu().numpy()
    errors = None
    if gt_file is not None:
        errors = compute_registration_error(data_dict['transform'], output_dict['estimated_transform'])
        print(f'RRE(deg): {errors[0]:.3f}, RTE(m): {errors[1]:.3f}')
    if output is not None:
        os.makedirs(output, exist_ok=True)
        np.save(os.path.join(output, 'estimated_transform.npy'), estimated_transform)
        ref_points = output_dict['ref_points'].cpu().numpy()
        src_points = output_dict['src_points'].cpu().numpy().astype(np.float64)
        aligned = src_points @ estimated_transform[:3, :3].T.astype(np.float64) + estimated_transform[:3, 3].astype(np.float64)
        ref_normals = src_normals = None
        if normals:
            ref_normals, src_normals = registration_normals(ref_points, output_dict['src_points'].cpu().numpy(), estimated_transform)
        write_ply(os.path.join(output, 'registration.ply'), ref_points, aligned, ref_normals, src_normals)
    return estimated_transform, errors


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    parser.add_argument('--src-file', required=True, help='src point cloud numpy file')
    parser.add_argument('--ref-file', required=True, help='ref point cloud numpy file')
    parser.add_argument('--gt-file', default=None, help='ground-truth transformation file')
    parser.add_argument('--weights', required=True, help='model weights file')
    parser.add_argument('--voxel-size', type=float, default=None, help='voxel-downsample both clouds first (Open3D semantics)')
    parser.add_argument('--output', default=None, help='directory for estimated_transform.npy and registration.ply')
    parser.add_argument('--normals', action='store_true', help='with --output: estimate normals (Open3D semantics) into the PLY')
    args = parser.parse_args(argv)
    if args.normals and args.output is None:
        parser.error('--normals needs --output')
    run(args.src_file, args.ref_file, args.weights, args.gt_file, args.voxel_size, args.output, args.normals)


if __name__ == '__main__':
    main()
