"""Generate tests/golden/lpips.npz: LPIPS and tLP100 of TecoGAN's two LPIPS copies, run unmodified with the seeded
AlexNet of synthetic.make_lpips_params(SEED), so that oracle/lpips.py and the device stay pinned to them on machines
without a reference checkout.

    python oracle/gen_lpips_golden.py [reference checkout, default $TECOGAN_REFERENCE or /root/reference]

- The official script (codes/official_metrics/metrics.py) runs in place through runpy, one process per run, on the
  PNG folders of the two sequences of tests/golden/official_metrics.npz (oracle/gen_official_metrics_golden.py), with
  its LPIPSmodels DistModel.  Stand-ins: skimage (compare_ssim is oracle.official_metrics.ssim), IPython.embed,
  matplotlib (imported, unused), the
  CUDA moves (the script asks for use_gpu=True; everything stays on the CPU, in fp32), torchvision.models.alexnet
  (the seeded features) and torch.load, which hands DistModel.initialize the seeded heads in place of those of
  weights/v0.1/alex.pth.
- MetricCalculator's DistModel (codes/metrics/LPIPS) with use_gpu=False and the same seeded weights scores the
  uncropped common-size frames of the same sequences through MetricCalculator.compute_LPIPS.

The file holds only numbers: per sequence k, lpips_k / tlp100_k (the script's per-frame lists) and calc_lpips_k
(MetricCalculator's per-frame LPIPS); the script's FrameAvg_*, FolderAvg_* and Avg_* of LPIPS and tLP100 over both.
"""
import os
import pickle
import subprocess
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SEED = 7
KEYS = ('LPIPS', 'tLP100')


def seeded_state_dict():
    import torch
    import synthetic
    return {k: torch.from_numpy(v) for k, v in synthetic.make_lpips_params(SEED).items()}


def _patch_alexnet():
    import torch
    import torchvision
    sd = seeded_state_dict()

    def alexnet(pretrained=False, **kw):
        m = torchvision.models.AlexNet()
        m.features.load_state_dict({k[len('features.'):]: v for k, v in sd.items() if k.startswith('features.')})
        return m
    torchvision.models.alexnet = alexnet
    return sd


def _heads(sd):
    return {k: v for k, v in sd.items() if k.startswith('lin')}


def install_stubs(codes):
    """Stand-ins for what both LPIPS copies import but do not use for a distance: skimage (compare_ssim is
    oracle.official_metrics.ssim), IPython.embed, matplotlib; and, for the reference's `codes` directory, the
    `metrics` package without its __init__ (as refimport.py does) and lmdb.  Idempotent."""
    from oracle import official_metrics as OM
    for name in ('skimage', 'skimage.measure', 'skimage.transform', 'skimage.color', 'IPython', 'matplotlib',
                 'matplotlib.pyplot', 'lmdb'):
        sys.modules.setdefault(name, types.ModuleType(name))
    for name in ('measure', 'transform', 'color'):
        setattr(sys.modules['skimage'], name, sys.modules['skimage.' + name])
    sys.modules['matplotlib'].pyplot = sys.modules['matplotlib.pyplot']
    sys.modules['skimage.measure'].compare_ssim = lambda x, y, data_range: OM.ssim(x, y, data_range)
    sys.modules['IPython'].embed = lambda *a, **k: None
    if codes not in sys.path:
        sys.path.insert(0, codes)
    m = types.ModuleType('metrics')            # skip metrics/__init__ (it imports the calculator's dependencies)
    m.__path__ = [os.path.join(codes, 'metrics')]
    sys.modules['metrics'] = m
    import scipy.signal
    import scipy.signal.windows
    if not hasattr(scipy.signal, 'gaussian'):  # utils/data_utils.py uses the removed alias
        scipy.signal.gaussian = scipy.signal.windows.gaussian


def _child_official(script, out_dir, results, targets, dump):
    import runpy
    import torch
    sd = _patch_alexnet()
    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.Tensor.cuda = lambda self, *a, **k: self
    install_stubs(os.path.dirname(os.path.dirname(os.path.abspath(script))))
    sys.path.insert(0, os.path.dirname(script))
    load = torch.load

    def load_seeded_heads(path, *a, **k):        # DistModel.initialize loads weights/v0.1/alex.pth: its heads
        heads = load(path, map_location="cpu")
        assert set(heads) == set(_heads(sd))
        return _heads(sd)
    torch.load = load_seeded_heads
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
    with open(dump, 'wb') as f:
        pickle.dump(res, f)


def calc_lpips(reference, true, pred):
    """MetricCalculator.compute_LPIPS of every frame pair, cropped to the common top-left size"""
    import torch
    sd = _patch_alexnet()
    install_stubs(os.path.join(reference, 'codes'))
    from metrics.metric_calculator import MetricCalculator
    from metrics.LPIPS.models.dist_model import DistModel
    dmod = DistModel()
    dmod.initialize(model='net-lin', net='alex', colorspace='rgb', spatial=False, use_gpu=False, gpu_ids=[0],
                    version='0.1')
    missing, unexpected = dmod.net.load_state_dict(_heads(sd), strict=False)
    assert not unexpected
    h, w = min(true.shape[1], pred.shape[1]), min(true.shape[2], pred.shape[2])
    out = []
    for t, p in zip(true, pred):
        ns = types.SimpleNamespace(true_img_cur=t[:h, :w], pred_img_cur=p[:h, :w], device=torch.device('cpu'),
                                   dm=dmod)
        out.append(MetricCalculator.compute_LPIPS(ns)[0, 0, 0, 0].item())
    return np.asarray(out, np.float64)


def official_pnetlin_lpips(reference, true, pred):
    """the official copy's PNetLin (codes/official_metrics/LPIPSmodels, unmodified, on the CPU in fp32) with the
    seeded weights on every frame pair, its inputs made by the copy's util.im2tensor as the script makes them"""
    sd = _patch_alexnet()
    install_stubs(os.path.join(reference, 'codes'))
    om = os.path.join(reference, 'codes', 'official_metrics')
    if om not in sys.path:
        sys.path.insert(0, om)
    from LPIPSmodels import networks_basic, util
    net = networks_basic.PNetLin(pnet_rand=False, pnet_tune=False, pnet_type='alex', use_dropout=True, use_gpu=False,
                                 spatial=False, version='0.1')
    missing, unexpected = net.load_state_dict(_heads(sd), strict=False)
    assert not unexpected and not missing
    net.eval()
    return np.asarray([float(net.forward(util.im2tensor(t), util.im2tensor(p)).flatten()[0])
                       for t, p in zip(true, pred)], np.float64)


def main(reference):
    from oracle import gen_official_metrics_golden as G
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'official_metrics.npz'))
    script = G.script_path(reference)
    arrays = {}
    with tempfile.TemporaryDirectory() as tmp:
        outs, tars = [], []
        for k in range(len(G.FOLDERS)):
            true, pred, (tar_dir, out_dir) = G.write_folders(tmp, k)
            assert np.array_equal(true, gold[f'true_{k}']) and np.array_equal(pred, gold[f'pred_{k}'])
            res = run(script, tmp, [out_dir], [tar_dir], f'folder{k}')
            arrays[f'lpips_{k}'] = np.asarray(res['list']['LPIPS'], np.float64)
            arrays[f'tlp100_{k}'] = np.asarray(res['list']['tLP100'], np.float64)
            arrays[f'calc_lpips_{k}'] = calc_lpips(reference, true, pred)
            outs.append(out_dir)
            tars.append(tar_dir)
        res = run(script, tmp, outs, tars, 'all')
    for name, v in res['totals'].items():
        arrays[name] = v
    arrays['seed'] = np.int64(SEED)
    path = os.path.join(ROOT, 'tests', 'golden', 'lpips.npz')
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path), 'bytes')


def run(script, tmp, results, targets, tag):
    dump = os.path.join(tmp, f'{tag}.pkl')
    out_dir = os.path.join(tmp, f'metrics_{tag}')
    subprocess.run([sys.executable, os.path.abspath(__file__), '--child', script, out_dir, ','.join(results),
                    ','.join(targets), dump], check=True, stdout=subprocess.DEVNULL)
    with open(dump, 'rb') as f:
        return pickle.load(f)


if __name__ == '__main__':
    if len(sys.argv) > 1 and sys.argv[1] == '--child':
        _child_official(*sys.argv[2:7])
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get('TECOGAN_REFERENCE', '/root/reference'))
