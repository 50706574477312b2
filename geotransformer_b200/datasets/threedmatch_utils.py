"""3DMatch / 3DLoMatch benchmark metadata: the gt.log / gt.info readers, the est.log writer and the transform error, with the names
and behaviour of ``geotransformer/datasets/registration/threedmatch/utils.py``.

A ``.log`` file is a sequence of 5-line records (``id0 id1 num_fragments``, then the 4 rows of the transform from fragment id1 to
fragment id0); a ``.info`` file a sequence of 7-line records (the same header, then the 6 x 6 covariance).  Values are read as
float32, as the reference does.  ``write_log_file`` writes ``transform.tolist()`` with Python's float formatting, tab-separated.
"""
import os

import numpy as np
import torch

from .. import functional as GF

# fragments per test scene of the 3DMatch benchmark
_NUM_FRAGMENTS = {
    '7-scenes-redkitchen': 60,
    'sun3d-home_at-home_at_scan1_2013_jan_1': 60,
    'sun3d-home_md-home_md_scan9_2012_sep_30': 60,
    'sun3d-hotel_uc-scan3': 55,
    'sun3d-hotel_umd-maryland_hotel1': 57,
    'sun3d-hotel_umd-maryland_hotel3': 37,
    'sun3d-mit_76_studyroom-76-1studyroom2': 66,
    'sun3d-mit_lab_hj-lab_hj_tea_nov_2_2012_scan1_erika': 38,
}
_ABBR = {
    '7-scenes-redkitchen': 'Kitchen',
    'sun3d-home_at-home_at_scan1_2013_jan_1': 'Home_1',
    'sun3d-home_md-home_md_scan9_2012_sep_30': 'Home_2',
    'sun3d-hotel_uc-scan3': 'Hotel_1',
    'sun3d-hotel_umd-maryland_hotel1': 'Hotel_2',
    'sun3d-hotel_umd-maryland_hotel3': 'Hotel_3',
    'sun3d-mit_76_studyroom-76-1studyroom2': 'Study',
    'sun3d-mit_lab_hj-lab_hj_tea_nov_2_2012_scan1_erika': 'MIT_Lab',
}


def get_num_fragments(scene_name):
    """Number of fragments of a 3DMatch test scene; ValueError for any other name."""
    try:
        return _NUM_FRAGMENTS[scene_name]
    except KeyError:
        raise ValueError(f'Unsupported test scene name "{scene_name}".') from None


def get_scene_abbr(scene_name):
    """Short scene name of the paper's tables (the name itself when it has none)."""
    return _ABBR.get(scene_name, scene_name)


def _read_records(file_name, rows, key):
    with open(file_name) as f:
        lines = [line.strip() for line in f.readlines()]
    records = []
    for start in range(0, len(lines) - len(lines) % (rows + 1), rows + 1):
        head = lines[start].split()
        body = np.array([lines[start + 1 + j].split() for j in range(rows)], dtype=np.float32)
        records.append({'test_pair': [int(head[0]), int(head[1])], 'num_fragments': int(head[2]), key: body})
    return records


def read_log_file(file_name):
    """Records ``{'test_pair': [id0, id1], 'num_fragments': n, 'transform': (4, 4) float32}`` of a .log file."""
    return _read_records(file_name, 4, 'transform')


def read_info_file(file_name):
    """Records ``{'test_pair': [id0, id1], 'num_fragments': n, 'covariance': (6, 6) float32}`` of a .info file."""
    return _read_records(file_name, 6, 'covariance')


def write_log_file(file_name, test_pairs):
    """Writes records with ``test_pair``, ``num_fragments`` and a (4, 4) ``transform`` as a .log file (creating its directory)."""
    directory = os.path.dirname(file_name)
    if directory:
        os.makedirs(directory, exist_ok=True)
    lines = []
    for pair in test_pairs:
        lines.append('{}\t{}\t{}\n'.format(pair['test_pair'][0], pair['test_pair'][1], pair['num_fragments']))
        lines.extend('{}\t{}\t{}\t{}\n'.format(*row) for row in pair['transform'].tolist())
    with open(file_name, 'w') as f:
        f.writelines(lines)


def get_gt_logs_and_infos(gt_root, num_fragments):
    """(gt_indices, gt_logs, gt_infos): gt_indices[id0, id1] = the record of the pair in gt.log, -1 for pairs not in it and for
    adjacent fragments (id1 <= id0 + 1), which the benchmark does not score."""
    gt_logs = read_log_file(os.path.join(gt_root, 'gt.log'))
    gt_infos = read_info_file(os.path.join(gt_root, 'gt.info'))
    gt_indices = np.full((num_fragments, num_fragments), -1, dtype=np.int32)
    for i, log in enumerate(gt_logs):
        id0, id1 = log['test_pair']
        if id1 > id0 + 1:
            gt_indices[id0, id1] = i
    return gt_indices, gt_logs, gt_infos


def compute_transform_error(transform, covariance, estimated_transform):
    """The 3DMatch realignment error ``er^T C er / C[0, 0]`` of ``estimated_transform`` against the gt ``transform`` with the gt.info
    ``covariance``, ``er = [t, q_xyz]`` of ``inv(transform) @ estimated_transform`` (q: nibabel's mat2quat, w >= 0).  Computed
    in double on the device (the current one for numpy inputs)."""
    device = next((x.device for x in (transform, covariance, estimated_transform) if isinstance(x, torch.Tensor)),
                  torch.device('cuda', torch.cuda.current_device()))

    def dev(x, n):
        t = x.detach() if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
        return t.to(device=device, dtype=torch.float32).reshape(1, n).contiguous()

    out = GF.registration_error_batched(dev(transform, 16), dev(estimated_transform, 16), covariances=dev(covariance, 36),
                                        rmse_threshold=0.0)
    return float(out[0, 2].item())
