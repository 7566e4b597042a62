"""Generate tests/golden/official_metrics.npz: per-frame PSNR / SSIM / tOF and the totals of TecoGAN's official
metric script (codes/official_metrics/metrics.py of a reference checkout), run unmodified on seeded PNG folders, so
that oracle/official_metrics.py and the device stay pinned to the script on machines without it.

    python oracle/gen_official_metrics_golden.py [reference checkout, default $TECOGAN_REFERENCE or /root/reference]

The script runs in place through runpy, one process per run (its absl flags cannot be defined twice in a process),
with stand-ins for what it imports but cannot run here: LPIPSmodels (a DistModel whose forward returns 0) and
skimage.measure.compare_ssim, which is oracle.official_metrics.ssim -- so the fixture's SSIM is oracle-derived.  Each
folder is scored alone (the script keeps per-frame float64 values only for its last folder) and then all folders
together for the totals.

The file holds, per folder k: true_k, pred_k (uint8 RGB [T, H, W, 3]; the target and output sizes differ) and
psnr_k, ssim_k, tof_k (float64, the script's per-frame lists); totals: FrameAvg_* / FolderAvg_* (the values the
script prints) and Avg_* (float32 per folder) for PSNR, SSIM and tOF; crop_n, crop_len, crop_off: the script's
crop_8x8 of n = 1 .. 2000 rows (length and offset of the slice it takes).
"""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ('PSNR', 'SSIM', 'tOF')
# (T, target h, w, output h, w): sizes that are not multiples of 32; folder 0's target is smaller than the output on
# one axis and larger on the other
FOLDERS = ((8, 100, 131, 104, 126), (7, 97, 130, 97, 130))


def script_path(reference):
    return os.path.join(reference, 'codes', 'official_metrics', 'metrics.py')


def folder_frames(k):
    import scipy.ndimage as nd
    T, ht, wt, hp, wp = FOLDERS[k]
    rng = np.random.default_rng(20 + k)
    h, w = max(ht, hp), max(wt, wp)
    base = nd.gaussian_filter(rng.uniform(0, 255, (h + 40, w + 40, 3)), (3.0, 3.0, 0))
    base = (base - base.min()) / (base.max() - base.min()) * 255
    full = np.stack([nd.shift(base, (0.9 * i, -1.4 * i, 0), order=1, mode='nearest')[20:20 + h, 20:20 + w]
                     for i in range(T)])
    full = np.clip(full, 0, 255).round()
    true = full[:, :ht, :wt].astype(np.uint8)
    pred = np.clip(full[:, :hp, :wp] + rng.integers(-10, 11, (T, hp, wp, 3)), 0, 255).astype(np.uint8)
    return true, pred


def _install_stubs():
    import types
    sys.path.insert(0, ROOT)
    from oracle import official_metrics as OM

    class DistModel:
        def initialize(self, **kw):
            pass

        def forward(self, a, b):
            return np.zeros(1)
    pkg = types.ModuleType('LPIPSmodels')
    util = types.ModuleType('LPIPSmodels.util')
    util.im2tensor = lambda img: img
    dm = types.ModuleType('LPIPSmodels.dist_model')
    dm.DistModel = DistModel
    pkg.util, pkg.dist_model = util, dm
    sk = types.ModuleType('skimage')
    skm = types.ModuleType('skimage.measure')
    skm.compare_ssim = lambda x, y, data_range: OM.ssim(x, y, data_range)
    sk.measure = skm
    sys.modules.update({'LPIPSmodels': pkg, 'LPIPSmodels.util': util, 'LPIPSmodels.dist_model': dm, 'skimage': sk,
                        'skimage.measure': skm})


def _child(script, out_dir, results, targets, dump):
    """one run of the unmodified script; dump its per-frame lists (last folder) and totals"""
    import runpy
    _install_stubs()
    argv, stdout = sys.argv, sys.stdout
    sys.argv = [script, f'--output={out_dir}', f'--results={results}', f'--targets={targets}']
    try:
        g = runpy.run_path(script, run_name='__main__')
    finally:
        sys.stdout, sys.argv = stdout, argv
    res = {'list': {k: [float(v) for v in g['list_dict'][k]] for k in KEYS}, 'totals': {}}
    for k in KEYS:
        res['totals']['FrameAvg_' + k] = np.asarray(g['sum_dict']['FrameAvg_' + k])[0]
        res['totals']['FolderAvg_' + k] = np.asarray(g['folder_dict']['FolderAvg_' + k])[0]
        res['totals']['Avg_' + k] = np.asarray(g['avg_dict']['Avg_' + k])
    crop = g['crop_8x8']
    res['crop'] = [(lambda img, y, x: (img.shape[0], y))(*crop(np.zeros((n, 1)))) for n in range(1, 2001)]
    with open(dump, 'wb') as f:
        pickle.dump(res, f)


def write_folders(tmp, k):
    import cv2
    true, pred = folder_frames(k)
    dirs = []
    for name, seq in (('tar', true), ('out', pred)):
        d = os.path.join(tmp, f'{name}_{k}')
        os.makedirs(d)
        for i, img in enumerate(seq):
            cv2.imwrite(os.path.join(d, f'col_res_{i:04d}.png'), img[..., ::-1])
        dirs.append(d)
    return true, pred, dirs


def run_script(script, tmp, results, targets, tag):
    dump = os.path.join(tmp, f'{tag}.pkl')
    out_dir = os.path.join(tmp, f'metrics_{tag}')
    subprocess.run([sys.executable, os.path.abspath(__file__), '--child', script, out_dir, ','.join(results),
                    ','.join(targets), dump], check=True, stdout=subprocess.DEVNULL)
    with open(dump, 'rb') as f:
        return pickle.load(f)


def main(reference):
    script = script_path(reference)
    arrays = {}
    with tempfile.TemporaryDirectory() as tmp:
        outs, tars = [], []
        for k in range(len(FOLDERS)):
            true, pred, (tar_dir, out_dir) = write_folders(tmp, k)
            arrays[f'true_{k}'], arrays[f'pred_{k}'] = true, pred
            res = run_script(script, tmp, [out_dir], [tar_dir], f'folder{k}')
            for key in KEYS:
                arrays[f'{key.lower()}_{k}'] = np.asarray(res['list'][key], np.float64)
            outs.append(out_dir)
            tars.append(tar_dir)
        res = run_script(script, tmp, outs, tars, 'all')
    for name, v in res['totals'].items():
        arrays[name] = v
    arrays['crop_n'] = np.arange(1, 2001)
    arrays['crop_len'] = np.asarray([c[0] for c in res['crop']])
    arrays['crop_off'] = np.asarray([c[1] for c in res['crop']])
    arrays['ssim_source'] = np.array('oracle.official_metrics.ssim standing in for skimage.measure.compare_ssim')
    path = os.path.join(ROOT, 'tests', 'golden', 'official_metrics.npz')
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    if len(sys.argv) > 1 and sys.argv[1] == '--child':
        _child(*sys.argv[2:7])
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get('TECOGAN_REFERENCE', '/root/reference'))
