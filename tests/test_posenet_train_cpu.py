"""PoseNet training without a GPU: the dropout rule's Philox against published vectors, the float64 reference
(tests/posenet_train_ref.py) against torch's autograd in double, and the new entry points' argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

import posenet_train_ref as T


def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32 with 10 rounds (also what curand_philox4x32_x.h computes on the host)."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
              (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in cases:
        got = tuple(int(v) for v in T.philox4x32_10(ctr, key))
        assert got == want, [hex(v) for v in got]
    # vectorised over counters = the scalar calls
    q = np.arange(5, dtype=np.uint64)
    vec = T.philox4x32_10((q, 0, 3, 7), (11, 13))
    for i in range(5):
        assert tuple(int(v[i]) for v in vec) == tuple(int(v) for v in T.philox4x32_10((i, 0, 3, 7), (11, 13)))


def test_dropout_multiplier_rule():
    seed = (0x123456789ABCDEF0, -5)
    assert np.all(T.dropout_multiplier(seed, 0, 10, 0.0) == 1) and np.all(T.dropout_multiplier(seed, 0, 10, 1.0) == 0)
    m = T.dropout_multiplier(seed, 1, 4099, 0.25)
    assert set(np.unique(m)) == {0.0, float(np.float32(1) / np.float32(0.75))}
    words = T.philox4x32_10((1024, 0, 1, (-5) & 0xFFFFFFFF), (0x9ABCDEF0, 0x12345678))   # elements 4096 .. 4099
    np.testing.assert_array_equal(m[4096:] > 0, np.array([int(w) for w in words])[:3] < int(0.75 * 2 ** 32))
    assert not np.array_equal(m, T.dropout_multiplier(seed, 2, 4099, 0.25))
    assert abs((m > 0).mean() - 0.75) < 5 * np.sqrt(0.75 * 0.25 / 4099)


class _FixedDropout(torch.nn.Module):
    """Stands in for a stage's nn.Dropout: multiplies by the injected masks in call order."""

    def __init__(self, masks):
        super().__init__()
        self.masks = list(masks)

    def forward(self, x):
        return x * self.masks.pop(0)


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_float64_reference_matches_torch_autograd(p):
    from pose2mesh_release_b200 import posenet

    J, H, S, B = 5, 24, 2, 9
    torch.manual_seed(3)
    net = posenet.LinearModel(J, H, S, p).double().train()
    g = torch.Generator().manual_seed(5)
    for name, t in net.state_dict().items():
        if "batch_norm" in name and t.dtype.is_floating_point:
            t.copy_(torch.rand(t.shape, generator=g, dtype=torch.float64) + 0.5)
    sd = {k: v.detach().clone().numpy() for k, v in net.state_dict().items()}
    masks = T.dropout_masks((17, 4), p, B, H, S)
    for s, st in enumerate(net.linear_stages):
        st.dropout = _FixedDropout(torch.from_numpy(m) for m in masks[2 * s:2 * s + 2])
    x = torch.randn(B, 2 * J, generator=g, dtype=torch.float64, requires_grad=True)
    d_out = torch.randn(B, 3 * J, generator=g, dtype=torch.float64)
    out = net(x)
    out.backward(d_out)
    val, bnd = T.forward_backward(sd, x.detach().numpy(), S, masks, d_out.numpy())
    tol = dict(rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(val["out"], out.detach().numpy(), **tol)
    np.testing.assert_allclose(val["dx"], x.grad.numpy(), **tol)
    n_grad = 0
    for name, prm in net.named_parameters():
        if prm.grad is None:                     # LinearModel.batch_norm1: constructed, never applied
            assert name.startswith("batch_norm1.")
            continue
        np.testing.assert_allclose(val["grad." + name], prm.grad.numpy(), err_msg=name, **tol)
        n_grad += 1
    assert n_grad == 4 + 8 * S
    after = net.state_dict()
    for name in val:
        if "running_" in name:
            np.testing.assert_allclose(val[name], after[name].numpy(), err_msg=name, **tol)
    assert all(np.all(np.isfinite(b)) and np.all(b >= 0) for b in bnd.values()) and set(bnd) == set(val)


def _host(*shape, dtype=np.float32):
    a = np.zeros(shape, dtype)
    return a, a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("name", ["p2m_posenet_train_forward", "p2m_posenet_backward"])
def test_train_entry_points_reject_host_arrays(name):
    """Like every stateless entry point: host memory in the data-array slots is P2M_ERR_INVALID naming the call, before
    any CUDA work.  Skipped with a GPU, where an entry point without the check would launch kernels on host pointers."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pose2mesh_release_b200 import _lib

    lib = _lib.load()
    B, J, H = 4, 4, 64
    keep = []

    def h(*shape, dtype=np.float32):
        a, p = _host(*shape, dtype=dtype)
        keep.append(a)
        return p

    params = _lib.PoseNetParams(num_joint=J, hidden=H, num_stage=0, w1_w=h(H, 2 * J), w1_b=h(H), w2_w=h(3 * J, H),
                                w2_b=h(3 * J))
    n_ws, n_sv = lib.p2m_posenet_train_workspace_bytes(B, J, H, 0), lib.p2m_posenet_train_saved_bytes(B, J, H, 0)
    assert n_ws > 0 and n_sv >= B * H * 4
    ws, sv, seed = h(n_ws, dtype=np.uint8), h(n_sv, dtype=np.uint8), h(2, dtype=np.int64)
    if name == "p2m_posenet_train_forward":
        extra = _lib.PoseNetTrain()
        args = (C.byref(params), C.byref(extra), h(B, 2 * J), B, 0.5, seed, h(B, 3 * J), h(B, J, 5), sv, n_sv, ws, n_ws)
    else:
        grads = _lib.PoseNetGrads(w1_w=h(H, 2 * J), w1_b=h(H), w2_w=h(3 * J, H), w2_b=h(3 * J))
        args = (C.byref(params), h(B, 2 * J), B, 0.5, seed, sv, n_sv, h(B, 3 * J), C.byref(grads), h(B, 2 * J), ws, n_ws)
    status = getattr(lib, name)(*args, None)
    msg = lib.p2m_last_error().decode()
    assert status == 1, (status, msg)
    assert name[len("p2m_"):] in msg and "device memory" in msg, msg
    # a batch of one has no batch statistics
    one = list(args)
    one[3 if name == "p2m_posenet_train_forward" else 2] = 1
    assert getattr(lib, name)(*one, None) == 1
    assert "more than one value per channel" in lib.p2m_last_error().decode()


def test_train_size_queries_return_zero_for_non_positive_sizes():
    from pose2mesh_release_b200 import _lib

    lib = _lib.load()
    for fn in (lib.p2m_posenet_train_workspace_bytes, lib.p2m_posenet_train_saved_bytes):
        assert fn(8, 17, 4096, 2) > 0 and fn(8, 17, 4096, 0) > 0
        for bad in ((0, 17, 4096, 2), (8, 0, 4096, 2), (8, 17, 0, 2), (8, 17, 4096, -1), (-3, 17, 4096, 2)):
            assert fn(*bad) == 0, bad
    # saved: (2 S + 1) [B, H] arrays and 8 S vectors of H
    assert lib.p2m_posenet_train_saved_bytes(256, 17, 4096, 2) == 5 * 256 * 4096 * 4 + 16 * 4096 * 4
