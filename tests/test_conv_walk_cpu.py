"""CPU tests (no GPU): the conv's walk-direction flag (TG_AMODE_REVERSE) in the header, the binding and the
argument check, and the walk directions FNet assigns along its chain of convs."""
import ctypes
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402,F401  (registers the package modules)

L = sys.modules['tecogan-pytorch_b200.lib']
N = sys.modules['tecogan-pytorch_b200.networks']


def test_reverse_flag_matches_header_and_leaves_the_a_modes_free():
    src = open(os.path.join(ROOT, 'include', 'tecogan_b200.h')).read()
    m = re.search(r'#define\s+TG_AMODE_REVERSE\s+(0x[0-9a-fA-F]+|\d+)', src)
    assert m and int(m.group(1), 0) == L.AMODE_REVERSE
    assert all(L.AMODE_REVERSE & mode == 0 for mode in (L.AMODE_AUTO, L.AMODE_HALO, L.AMODE_TAP))


def test_conv_checks_the_a_mode_under_the_reverse_flag_without_a_gpu():
    lib = L.load()
    d = L.ConvDesc()
    d.x = d.weights = d.bias = d.y = 16
    d.n, d.h, d.w, d.cin, d.cout, d.act = 1, 8, 8, 64, 64, L.ACT_RELU
    d.a_mode = 3 | L.AMODE_REVERSE
    assert lib.tg_conv_tcgen05(ctypes.byref(d), None) == -1 and b'a_mode' in lib.tg_last_error_string()
    d.a_mode = 0x200
    assert lib.tg_conv_tcgen05(ctypes.byref(d), None) == -1 and b'a_mode' in lib.tg_last_error_string()


def test_fnet_chain_alternates_over_every_conv_in_execution_order():
    net = N.FNet(3)
    mods = [m for m, _, _ in net.conv_layers(64, 64)]
    chain = sorted(N.FNet.CHAIN, key=N.FNet.CHAIN.get)
    assert [getattr(net, b)[i] for b, i in chain] == mods
    # encoder1[0] and flow[0] read the reversed walks of pack_pair and upsample2x: both walk forward
    assert N.FNet.CHAIN[('encoder1', 0)] % 2 == 0 and N.FNet.CHAIN[('flow', 0)] % 2 == 0
    assert N.FNet.CHAIN[('flow', 2)] % 2 == 1
