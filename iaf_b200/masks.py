"""Host-side AR masks (numpy).  The device builds its own masks inside the pack kernel
(csrc/iaf_pack.cu); these are for host logic that needs them as arrays: ``postup`` and
parameter initialisation.  Rules: tf_utils/layers.py:115-141, graphy/nodes/ar.py:241-264."""
import numpy as np


def centre_visible(n_in, n_out, zerodiagonal):
    """[n_in, n_out] MADE mask of the centre tap."""
    ci = np.arange(n_in)[:, None]
    co = np.arange(n_out)[None, :]
    if n_out >= n_in:
        assert n_out % n_in == 0
        grp = co // (n_out // n_in)
        vis = ci < grp if zerodiagonal else ci <= grp
    else:
        assert n_in % n_out == 0
        k = n_in // n_out
        vis = ci < co * k if zerodiagonal else ci < (co + 1) * k
    return vis.astype(np.float32)


def tf_conv_ar_mask(n_in, n_out, zerodiagonal):
    """[3,3,n_in,n_out]."""
    m = np.zeros((3, 3, n_in, n_out), np.float32)
    m[1, 2] = 1
    m[2] = 1
    m[1, 1] = centre_visible(n_in, n_out, zerodiagonal)
    return m


def theano_conv_ar_mask(n_in, n_out, size_kernel=(3, 3), zerodiagonal=True, flipmask=False):
    """[n_out, n_in+1, 3, 3] including the pad channel (never sees the centre tap).  flipmask: the mask reversed on all
    four axes, pad channel included (ar.py:263-264); the pad channel then inherits channel 0's centre column."""
    assert tuple(size_kernel) == (3, 3)
    m = np.zeros((n_out, n_in + 1, 3, 3), np.float32)
    m[:, :, 1, 2] = 1
    m[:, :, 2, :] = 1
    m[:, :n_in, 1, 1] = centre_visible(n_in, n_out, zerodiagonal).T
    if flipmask:
        m = np.ascontiguousarray(m[::-1, ::-1, ::-1, ::-1])
    return m
