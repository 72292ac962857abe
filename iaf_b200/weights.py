"""Weight import for the IAF operator (SURVEY 8f-3): the two parameter containers the reference
writes, mapped onto IAFOperator.set_weights() triples.

* Theano: ``<dir>/weights.ndict.tar.gz`` = ``arrays.npz`` (positional ``arr_i``) + ``names.txt`` (sorted keys),
  graphy/ndict.py:209-236, loaded by train.py:133-138.  IAF parameters are named
  ``{i}_{j}_posterior_conv1_{k}_{w,b,s}`` / ``{i}_{j}_posterior_conv1_out_{k}_{w,b,s}`` (models.py:410,92; ar.py:388-394,288-296).
* TF: variables ``model/IAF_{i}_{j}/ar_multiconv2d/layer_{k}/{V,g,b}`` and ``.../layer_out_{k}/{V,g,b}``
  (tf_train.py:186,69; layers.py:160-166,53-55), e.g. exported from a checkpoint to an .npz keyed by variable name.
"""
import io
import tarfile

import numpy as np
import torch


def _as_f32(a, device):
    if torch.is_tensor(a):
        return a.detach().to(torch.float32).contiguous().to(device)
    return torch.as_tensor(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).to(device)


def np_loadz(filename):
    """Read a graphy ``.ndict.tar.gz`` (graphy/ndict.py:228-236) -> dict name -> ndarray."""
    with tarfile.open(filename, "r:gz") as tar:
        members = {m.name: m for m in tar.getmembers()}
        arrays = np.load(io.BytesIO(tar.extractfile(members["arrays.npz"]).read()))
        names = tar.extractfile(members["names.txt"]).read().decode().splitlines()
        return {names[i]: arrays["arr_%d" % i] for i in range(len(names))}


def np_savez(d, filename):
    """Write the same container (graphy/ndict.py:209-226): keys sorted, arrays positional."""
    keys = sorted(d)
    buf = io.BytesIO()
    np.savez(buf, *[np.asarray(d[k]) for k in keys])
    txt = ("".join("%s\n" % k for k in keys)).encode()
    with tarfile.open(filename, "w:gz") as tar:
        for name, data in (("arrays.npz", buf.getvalue()), ("names.txt", txt)):
            ti = tarfile.TarInfo(name)
            ti.size = len(data)
            tar.addfile(ti, io.BytesIO(data))


def theano_layers(w, name, n_hidden, n_heads=2, device="cuda"):
    """(w, s, b) triples, hidden layers first, for ``multiconv2d(name, ...)`` parameters in ``w``."""
    names = ["%s_%d" % (name, i) for i in range(n_hidden)] + ["%s_out_%d" % (name, k) for k in range(n_heads)]
    t = lambda a: _as_f32(a, device)
    return [(t(w[n + "_w"]), t(w[n + "_s"]), t(w[n + "_b"])) for n in names]


def deinterleave_heads(w, s, b):
    """The two heads of a linear IAF conv ``ar.conv2d(name, n_z, 2 n_z)`` (models.py:55-56, 79-82): its output rows
    interleave them, ``mean = out[:, ::2]``, ``logsd = out[:, 1::2]`` (models.py:152-161, 246-259).  Returns the
    (w, s, b) triples of the mean and the logsd head, views of the given tensors (so autograd scatters their gradients
    back into the interleaved rows).  Row 2i and row 2i + 1 have the mask of row i of ``ar.conv2d(n_z, n_z)`` with
    zerodiagonal (ar.py:250-256), and weight normalisation is per row, so each head is an ordinary heads conv."""
    return [(w[k::2], s[k::2], b[k::2]) for k in range(2)]


def tf_layers(variables, scope, n_hidden=2, n_heads=2, device="cuda"):
    """(V, g, b) triples for ``ar_multiconv2d`` under ``scope`` (e.g. ``model/IAF_0_3/ar_multiconv2d``)."""
    names = ["layer_%d" % i for i in range(n_hidden)] + ["layer_out_%d" % k for k in range(n_heads)]
    t = lambda a: _as_f32(a, device)
    return [tuple(t(variables["%s/%s/%s" % (scope, n, k)]) for k in "Vgb") for n in names]
