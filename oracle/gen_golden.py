"""Generate tests/golden/*.npz by running the UNMODIFIED reference
(skycrapers/TecoGAN-PyTorch @ 903b070, installed into oracle/_ref by build()) on seeded inputs:

    python oracle/gen_golden.py            # all fixtures
    python oracle/gen_golden.py full       # only the full-size sample

Import recipe = SURVEY.md section 9 (two module stubs, no edits to the reference).
Inputs and weights are NOT stored: they are regenerated from seeds by
oracle.frnet_oracle.make_frnet_params / numpy default_rng, so the fixtures hold
only the reference's outputs.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def import_reference():
    import refimport                                        # SURVEY.md section 9 recipe, no reference edits
    return refimport.import_generator()


def rand(seed, *shape, lo=0.0, hi=1.0):
    return torch.from_numpy(np.random.default_rng(seed).uniform(lo, hi, size=shape).astype(np.float32))


def gen_downsample_bd(data_utils, out_dir):
    """BD degradation of the data side (SURVEY 8-f2): create_kernel + downsample_bd
    (codes/utils/data_utils.py:11-53) -- the reference calls scipy.signal.gaussian, an alias that
    newer scipy only keeps under scipy.signal.windows."""
    import scipy.signal
    if not hasattr(scipy.signal, 'gaussian'):
        scipy.signal.gaussian = scipy.signal.windows.gaussian
    kern = data_utils.create_kernel(1.5)                      # [3,3,9,9]
    a = data_utils.downsample_bd(rand(30, 2, 3, 36, 44), kern, 4, pad_data=True)
    b = data_utils.downsample_bd(rand(31, 1, 3, 41, 45), kern, 4, pad_data=False)
    c = data_utils.downsample_bd(rand(32, 1, 3, 27, 30), kern, 2, pad_data=True)
    np.savez_compressed(os.path.join(out_dir, 'downsample_bd.npz'), kernel=kern.numpy(),
                        s4_pad=a.numpy(), s4_valid=b.numpy(), s2_pad=c.numpy())


GRAD_FULL = ('fnet.encoder1.0.weight', 'fnet.flow.2.weight', 'fnet.flow.2.bias', 'srnet.conv_in.0.weight',
             'srnet.resblocks.1.conv.2.bias', 'srnet.conv_up.2.bias', 'srnet.conv_out.weight', 'srnet.conv_out.bias')


def gen_full_size_sample(FRNet, out_dir):
    """FRNet.step at the bench size (1 clip, 3x134x320 -> 536x1280, 2x weights): the full frame is 8 MB, so a
    fixed, seeded sample of 65536 output values is stored with its flat indices."""
    from oracle.frnet_oracle import make_frnet_params
    net = FRNet(3, 3, 64, 10, 'BD', 4)
    net.load_state_dict(make_frnet_params(5, gain=2.0), strict=True)
    net.eval()
    lr_curr, lr_prev, hr_prev = rand(1, 1, 3, 134, 320), rand(2, 1, 3, 134, 320), rand(3, 1, 3, 536, 1280)
    with torch.no_grad():
        hr = net.step(lr_curr, lr_prev, hr_prev).numpy().reshape(-1)
    idx = np.sort(np.random.default_rng(0).choice(hr.size, size=1 << 16, replace=False))
    np.savez_compressed(os.path.join(out_dir, 'step_bd4_134x320_g2_sample.npz'), index=idx.astype(np.int64),
                        hr_curr=hr[idx].astype(np.float32))


def gen_sequence_grads(FRNet, out_dir):
    from oracle.frnet_oracle import make_frnet_params
    net = FRNet(3, 3, 64, 2, 'BD', 4)
    net.load_state_dict(make_frnet_params(15, nb=2, scale=4, degradation='BD', gain=1.5), strict=True)
    net.train()
    lr_data = rand(9, 1, 3, 3, 16, 16).requires_grad_(True)
    d = net.forward_sequence(lr_data)
    rng = np.random.default_rng(16)
    r1 = torch.from_numpy(rng.uniform(-1, 1, size=tuple(d['hr_data'].shape)).astype(np.float32))
    r2 = torch.from_numpy(rng.uniform(-1, 1, size=tuple(d['lr_flow'].shape)).astype(np.float32))
    loss = (d['hr_data'] * r1).sum() + 0.05 * (d['lr_flow'] * r2).sum()
    loss.backward()
    named = dict(net.named_parameters())
    out = {'loss': np.float32(loss.item()), 'd_lr_data': lr_data.grad.numpy(),
           'names': np.array(list(named)), 'norms': np.array([float(v.grad.norm()) for v in named.values()], np.float64)}
    for k in GRAD_FULL:
        out['g:' + k] = named[k].grad.numpy()
    np.savez_compressed(os.path.join(out_dir, 'fwd_seq_grads_bd4_16x16_nb2_g15.npz'), **out)
    print('sequence grads: loss', loss.item(), 'max |d lr_data|', float(lr_data.grad.abs().max()))


def main():
    from oracle.frnet_oracle import make_frnet_params, make_clip
    FRNet, net_utils, data_utils = import_reference()
    out_dir = os.path.join(ROOT, 'tests', 'golden')
    os.makedirs(out_dir, exist_ok=True)
    torch.set_num_threads(8)
    gen_downsample_bd(data_utils, out_dir)
    if sys.argv[1:] == ['bd']:                       # only this fixture
        return
    if sys.argv[1:] == ['grads']:
        return gen_sequence_grads(FRNet, out_dir)
    if sys.argv[1:] == ['full']:
        return gen_full_size_sample(FRNet, out_dir)

    def ref_model(scale, degradation, seed, gain, nb=10):
        net = FRNet(3, 3, 64, nb, degradation, scale)
        sd = make_frnet_params(seed, nb=nb, scale=scale, degradation=degradation, gain=gain)
        net.load_state_dict(sd, strict=True)
        return net.eval()

    # ---- 1. FRNet.step, 4x BD, size not a multiple of 8 (reflect pad 2 rows / 4 cols)
    for tag, gain in (('g1', 1.0), ('g15', 1.5), ('g2', 2.0)):
        net = ref_model(4, 'BD', seed=11, gain=gain)
        lr_curr, lr_prev = rand(1, 1, 3, 18, 28), rand(2, 1, 3, 18, 28)
        hr_prev = rand(3, 1, 3, 72, 112)
        with torch.no_grad():
            lr_flow = net.fnet(lr_curr, lr_prev)
            hr = net.step(lr_curr, lr_prev, hr_prev)
        np.savez_compressed(os.path.join(out_dir, f'step_bd4_18x28_{tag}.npz'),
                            lr_flow=lr_flow.numpy(), hr_curr=hr.numpy(),
                            meta=np.array([4, 11, 1, 2, 3], dtype=np.int64), gain=np.float32(gain))
        print(tag, 'flow absmax', float(lr_flow.abs().max()), 'hr range', float(hr.min()), float(hr.max()))

    # ---- 2. FRNet.step, 2x BI (bilinear upsample_func), pad 4 rows
    net = ref_model(2, 'BI', seed=12, gain=1.5)
    lr_curr, lr_prev = rand(4, 1, 3, 20, 24), rand(5, 1, 3, 20, 24)
    hr_prev = rand(6, 1, 3, 40, 48)
    with torch.no_grad():
        lr_flow = net.fnet(lr_curr, lr_prev)
        hr = net.step(lr_curr, lr_prev, hr_prev)
    np.savez_compressed(os.path.join(out_dir, 'step_bi2_20x24_g15.npz'),
                        lr_flow=lr_flow.numpy(), hr_curr=hr.numpy(), gain=np.float32(1.5))

    # ---- 3. FRNet.infer_sequence (uint8 THWC), 4x BD, 4 frames of a moving clip
    net = ref_model(4, 'BD', seed=13, gain=1.5)
    clip = make_clip(7, 4, 3, 16, 24)
    with torch.no_grad():
        seq = net.infer_sequence(clip, torch.device('cpu'))
    np.savez_compressed(os.path.join(out_dir, 'infer_seq_bd4_16x24_g15.npz'), hr_seq=seq)
    print('infer_sequence', seq.shape, seq.dtype)

    # ---- 4. FRNet.forward_sequence (training forward), 4x BD, n=1 t=3 16x16
    net = ref_model(4, 'BD', seed=14, gain=1.5)
    lr_data = rand(8, 1, 3, 3, 16, 16)
    net.train()
    with torch.no_grad():
        d = net.forward_sequence(lr_data)
    np.savez_compressed(os.path.join(out_dir, 'fwd_seq_bd4_16x16_g15.npz'),
                        **{k: v.numpy() for k, v in d.items()})

    # ---- 4b. gradients of forward_sequence (generator backward, SURVEY 8-f1), nb=2 to keep it small:
    # loss = <hr_data, R1> + 0.05 <lr_flow, R2>; stored: loss, d/d lr_data, a few whole parameter
    # gradients and the L2 norm of every parameter gradient
    gen_sequence_grads(FRNet, out_dir)
    gen_full_size_sample(FRNet, out_dir)

    # ---- 5. functional ops
    x = rand(20, 2, 3, 20, 24)
    flow = rand(21, 2, 2, 20, 24, lo=-4.0, hi=4.0)
    flow[0, :, 0, 0] = torch.tensor([-30.0, 40.0])   # far out of range -> border clamp
    warped = net_utils.backward_warp(x, flow)
    s2d4 = net_utils.space_to_depth(rand(22, 2, 3, 16, 24), 4)
    s2d2 = net_utils.space_to_depth(rand(22, 2, 3, 16, 24), 2)
    bic4 = net_utils.BicubicUpsampler(4)(rand(23, 1, 3, 9, 11))
    bic2 = net_utils.BicubicUpsampler(2)(rand(23, 1, 3, 9, 11))
    bil4 = net_utils.get_upsampling_func(4, 'BI')(rand(23, 1, 3, 9, 11))
    bil2 = net_utils.get_upsampling_func(2, 'BI')(rand(23, 1, 3, 9, 11))
    q_in = np.concatenate([np.arange(-3, 520, dtype=np.float32) / np.float32(510.0),   # x.5 ties
                           np.random.default_rng(24).uniform(-0.2, 1.2, 1000).astype(np.float32)])
    q = data_utils.float32_to_uint8(q_in)
    convt = torch.nn.ConvTranspose2d(8, 8, 3, 2, 1, output_padding=1)
    wt = rand(25, 8, 8, 3, 3, lo=-1, hi=1)
    bt = rand(26, 8, lo=-1, hi=1)
    with torch.no_grad():
        convt.weight.copy_(wt)
        convt.bias.copy_(bt)
        ct = convt(rand(27, 1, 8, 5, 7))
    np.savez_compressed(os.path.join(out_dir, 'ops.npz'),
                        warped=warped.numpy(), s2d4=s2d4.numpy(), s2d2=s2d2.numpy(),
                        bic4=bic4.numpy(), bic2=bic2.numpy(), bil4=bil4.numpy(), bil2=bil2.numpy(),
                        q_in=q_in, q=q, convt=ct.numpy())
    print('done ->', out_dir)


if __name__ == '__main__':
    main()
