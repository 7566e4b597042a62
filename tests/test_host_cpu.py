"""CPU tests (no GPU, no compute calls): the C-ABI library loads and exports every symbol the
header declares; the Python host mirrors the reference's module surface; clip sharding over
world_size-2 gloo."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
from oracle import frnet_oracle as O           # noqa: E402

L = sys.modules['tecogan-pytorch_b200.lib']


def header_symbols():
    src = open(os.path.join(ROOT, 'include', 'tecogan_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(tg_[a-zA-Z0-9_]+)\s*\(', src)))


def test_library_exports_every_header_symbol():
    assert os.path.isfile(L.LIB_PATH), 'build the library first: python -c "import __graft_entry__ as g; g.build()"'
    lib = ctypes.CDLL(L.LIB_PATH)
    names = header_symbols()
    assert len(names) >= 19
    for name in names:
        assert hasattr(lib, name), f'{name} declared in include/tecogan_b200.h but not exported'
    # the ctypes binding covers exactly the header
    assert sorted(L.exported_symbols()) == names
    T.load_library()
    assert L.load().tg_version() == 2          # ABI 2: tg_conv_desc.mask + the backward entry points
    assert L.load().tg_packed_weight_bytes(64, 64) == 9 * 64 * 128
    assert L.load().tg_packed_weight_bytes(256, 256) == 9 * 4 * 256 * 128
    assert L.load().tg_packed_weight_bytes(60, 64) == 0


def test_conv_desc_struct_layout_matches_header():
    # 5 pointers + 12 int32 + the mask pointer (see struct tg_conv_desc)
    assert ctypes.sizeof(L.ConvDesc) == 5 * 8 + 12 * 4 + 8
    assert L.ConvDesc.n.offset == 40 and L.ConvDesc.max_ctas.offset == 40 + 10 * 4
    assert L.ConvDesc.mask.offset == 88
    # struct tg_wgrad_desc: 5 pointers + 10 int32
    assert ctypes.sizeof(L.WgradDesc) == 5 * 8 + 10 * 4 and L.WgradDesc.n.offset == 40


def test_backward_entry_points_reject_bad_arguments_without_a_gpu():
    lib = L.load()
    assert lib.tg_grad_scale_workspace_bytes() == 16
    w = L.WgradDesc()
    assert lib.tg_wgrad_tcgen05(ctypes.byref(w), None) == -1 and b'null' in lib.tg_last_error_string()
    w.x = w.dz = w.dw = 16
    w.n, w.h, w.w, w.cin, w.cout, w.cin_real, w.cout_real = 1, 8, 8, 48, 64, 48, 64
    assert lib.tg_wgrad_tcgen05(ctypes.byref(w), None) == -2                    # stored cin must be 64/128/256
    d = L.ConvDesc()
    d.x = d.weights = d.bias = d.y = 16
    d.n, d.h, d.w, d.cin, d.cout, d.act = 1, 8, 8, 64, 64, L.ACT_DRELU
    assert lib.tg_conv_tcgen05(ctypes.byref(d), None) == -1 and b'mask' in lib.tg_last_error_string()
    assert lib.tg_upsample_bwd_nchw_f32(ctypes.c_void_p(16), ctypes.c_void_p(16), 1, 2, 8, 8, 3, 0, 1.0, 0, None) == -2
    assert lib.tg_warp_s2d_concat_bwd(None, None, None, None, None, None, 1, 3, 8, 8, 4, 64, None) == -1


def test_null_and_bad_arguments_are_rejected_without_a_gpu():
    lib = L.load()
    rc = lib.tg_maxpool2x2_nhwc_f16(None, None, 1, 4, 4, 64, None)
    assert rc == -1 and b'null' in lib.tg_last_error_string()
    rc = lib.tg_warp_s2d_concat_hrflow(ctypes.c_void_p(16), ctypes.c_void_p(16), ctypes.c_void_p(16),
                                       ctypes.c_void_p(16), 1, 3, 8, 8, 3, 64, None)
    assert rc == -2 and b'scale' in lib.tg_last_error_string()
    d = L.ConvDesc()
    assert lib.tg_conv_tcgen05(ctypes.byref(d), None) == -1
    d.x = d.weights = d.bias = d.y = 16
    d.n, d.h, d.w, d.cin, d.cout = 1, 8, 8, 48, 64
    assert lib.tg_conv_tcgen05(ctypes.byref(d), None) == -2      # cin must be 64/128/256
    d.cin, d.cin_real = 64, 65                                   # real input channels beyond the stored ones
    assert lib.tg_conv_tcgen05(ctypes.byref(d), None) == -1 and b'cin_real' in lib.tg_last_error_string()
    assert L.ConvDesc.cin_real.offset == 40 + 11 * 4             # the former `reserved` slot: layout unchanged
    with pytest.raises(L.TecoganB200Error):
        L.check(-2, 'tg_conv_tcgen05')


@pytest.mark.parametrize('scale,deg', [(4, 'BD'), (4, 'BI'), (2, 'BD'), (2, 'BI')])
def test_state_dict_is_reference_compatible(scale, deg):
    net = T.FRNet(3, 3, 64, 10, deg, scale)
    shapes = O.frnet_param_shapes(scale=scale, degradation=deg)
    sd = net.state_dict()
    assert list(sd.keys()) == list(shapes.keys())          # same keys, same ORDER as the reference
    for k, v in sd.items():
        assert tuple(v.shape) == tuple(shapes[k]), k
    net.load_state_dict(O.make_frnet_params(1, scale=scale, degradation=deg), strict=True)
    if deg == 'BD':
        assert torch.equal(net.upsample_func.kernels, net.srnet.upsample_func.kernels)
        from oracle.ops_oracle import bicubic_kernels
        assert np.array_equal(T.BicubicUpsampler(scale).kernels.numpy(), bicubic_kernels(scale))


@pytest.mark.parametrize('nc,scale', [(1, 4), (2, 4), (3, 4), (4, 2), (12, 2)])
def test_frnet_accepts_channel_counts_its_kernels_run(nc, scale):
    """(scale^2 + 1) * nc SRNet input channels fit the 64-channel map: 17 / 34 / 51 at 4x, 20 / 60 at 2x"""
    net = T.FRNet(nc, nc, 64, 1, 'BD', scale)
    assert net.fnet.in_nc == nc and net.srnet.conv_in[0].in_channels == (scale ** 2 + 1) * nc
    assert net.srnet.conv_out.out_channels == nc
    net.load_state_dict(O.make_frnet_params(1, in_nc=nc, out_nc=nc, nb=1, scale=scale), strict=True)


@pytest.mark.parametrize('in_nc,out_nc,scale,match', [
    (3, 1, 4, r'in_nc=3 != out_nc=1'), (1, 3, 2, r'in_nc=1 != out_nc=3'),
    (4, 4, 4, r'= 68 SRNet input channels .* at most 64'), (13, 13, 2, r'= 65 SRNet input channels .* at most 64')])
def test_frnet_refuses_channel_counts_no_kernel_runs(in_nc, out_nc, scale, match):
    with pytest.raises(T.TecoganB200Error, match=match):
        T.FRNet(in_nc, out_nc, 64, 1, 'BD', scale)


def test_profile_matches_reference_counter():
    net = T.FRNet(3, 3, 64, 10, 'BD', 4)
    g, p = net.profile((3, 134, 320))
    assert list(g.keys()) == ['FNet', 'SRNet']
    assert abs(g['FNet'] - 10.511) < 1e-3 and abs(g['SRNet'] - 83.927) < 1e-3   # SURVEY.md 0.6
    assert p['FNet'] == 1745506 and p['SRNet'] == 843587
    g2, _ = T.FRNet(3, 3, 64, 10, 'BI', 2).profile((3, 268, 640))
    assert abs(g2['FNet'] - 43.019) < 1e-3 and abs(g2['SRNet'] - 270.897) < 1e-3


def test_define_generator_and_error_behaviour():
    opt = {'scale': 4, 'dataset': {'degradation': {'type': 'BD'}},
           'model': {'generator': {'name': 'FRNet', 'in_nc': 3, 'out_nc': 3, 'nf': 64, 'nb': 10}}}
    net = T.define_generator(opt)
    assert isinstance(net, T.FRNet) and net.scale == 4
    opt['model']['generator']['name'] = 'nope'
    with pytest.raises(ValueError, match='Unrecognized generator'):
        T.define_generator(opt)
    with pytest.raises(ValueError, match='Unrecognized degradation'):
        T.get_upsampling_func(4, 'XX')
    # no CPU fallback: CPU tensors are refused loudly
    with pytest.raises(T.TecoganB200Error):
        net.step(torch.zeros(1, 3, 8, 8), torch.zeros(1, 3, 8, 8), torch.zeros(1, 3, 32, 32))
    with pytest.raises(T.TecoganB200Error):
        T.space_to_depth(torch.zeros(1, 3, 8, 8), 4)
    data = net.generate_dummy_data((3, 16, 24), torch.device('cpu'))
    assert [tuple(t.shape) for t in data] == [(1, 3, 16, 24), (1, 3, 16, 24), (1, 3, 64, 96)]


def test_yaml_configs_of_the_reference_surface_parse():
    import yaml
    y = yaml.safe_load('''
scale: 4
dataset: {degradation: {type: BD, sigma: 1.5}}
model:
  name: TecoGAN
  generator: {name: FRNet, in_nc: 3, out_nc: 3, nf: 64, nb: 10, load_path: ~}
''')
    assert isinstance(T.define_generator(y), T.FRNet)


def test_clip_sharding_single_process():
    assert T.clips_for_rank(10, 1, 4) == [1, 5, 9]
    allc = sorted(sum((T.clips_for_rank(11, r, 4) for r in range(4)), []))
    assert allc == list(range(11))
    with pytest.raises(ValueError):
        T.clips_for_rank(4, 4, 4)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    mine = T.clips_for_rank(7, rank, world)
    # the bench's reduction: frames processed summed, elapsed time max over ranks
    frames = torch.tensor([float(len(mine) * 10)])
    elapsed = torch.tensor([1.0 + rank])
    dist.all_reduce(frames, op=dist.ReduceOp.SUM)
    dist.all_reduce(elapsed, op=dist.ReduceOp.MAX)
    gathered = [None] * world
    dist.all_gather_object(gathered, mine)
    q.put((rank, gathered, float(frames), float(elapsed)))
    dist.barrier()
    dist.destroy_process_group()


def test_clip_sharding_world_size_2_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 1000)
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, gathered, frames, elapsed in res:
        assert sorted(gathered[0] + gathered[1]) == list(range(7))      # disjoint cover
        assert set(gathered[0]).isdisjoint(gathered[1])
        assert frames == 70.0 and elapsed == 2.0                         # sum of work, max of time


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` is the arm the driver times beside ours; it runs on the host cores
    (no GPU needed) and must print ONE JSON line with the contract's keys; under torchrun only rank 0
    works and prints."""
    import json
    import subprocess
    env = dict(os.environ)
    env.pop('RANK', None)
    cmd = [sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '1']
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-800:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ('impl', 'metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better',
              'scaling', 'vs_baseline', 'dtype', 'data', 'config', 'cpu_baseline', 'e2e', 'gpu_launches'):
        assert k in d, k
    assert d['impl'] == 'reference' and d['value'] > 0 and d['higher_is_better'] is True
    import refimport
    assert d['cpu_baseline']['kind'] == ('reference' if refimport.available() else 'port') and d['cpu_baseline']['cores'] >= 1
    assert d['config']['clips_per_gpu'] == 4          # the same 4-clip step as the GPU arm
    assert d['e2e'] == {'value': d['value'], 'unit': d['unit'], 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}
    # a non-zero rank exits 0 without work or output
    env.update(RANK='1', WORLD_SIZE='2', LOCAL_RANK='1')
    out = subprocess.run(cmd[:-4] + ['--gpus', '2', '--steps', '1', '--warmup', '1'], capture_output=True, text=True,
                         timeout=120, env=env, cwd=ROOT)
    assert out.returncode == 0 and out.stdout.strip() == ''
