"""The max-pooling kernels (``bns_sage_max_f32``, ``bns_sage_max_bwd_f32``, ``bns_sage_max_infer_f32`` and its block
variant) against the restatement of tests/sage_pool_reference.py, on GAT's crafted partition graph: an empty row, rows
of degree 1 to 33, a 4100-entry row full of repeated sources (multi-edges), halo-only rows, rows whose halo entries are
all unsampled, and a row whose halo chunks hold 0 to 33 sampled entries.  ``y`` takes values on a grid of quarters, so
equal nonzero values from different sources are common, and a few columns are all zero after the ReLU.  A max involves
no rounding: ``m`` and the winners must be exact; ``d y`` sums in transposed-CSR order and is held to float64 at
1e-6."""
import pytest
import torch

from tests.sage_pool_reference import sage_max_backward_reference, sage_max_reference
from tests.test_gat_train_attention_gpu import N_IN, R_EMPTY, R_LONG, _crafted

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
WIDTHS = (4, 44, 128, 256, 604, 1024)


def _y(n, Fp, seed):
    gen = torch.Generator().manual_seed(seed)
    y = torch.round(torch.randn(n, Fp, generator=gen) * 4) / 4
    y[:, :Fp:7] = -1.0                                      # all-zero columns of z
    return y


def _forward(g, y, halo=True):
    """The raw forward kernel: ``(m, win)``."""
    from bns_gcn_b200._lib import check, lib
    z = torch.relu(y).contiguous()
    n_in, Fp = g.n_in, z.shape[1]
    m = torch.empty(n_in, Fp, device=DEV)
    win = torch.empty(n_in, Fp, dtype=torch.int32, device=DEV)
    c = g.compact if halo else None
    check(lib.bns_sage_max_f32(g.a_in._h, None if c is None else g.a_out._h, None if c is None else c.cidx.data_ptr(),
                               None if c is None else c.chunk_cnt.data_ptr(), None if c is None else c.cpos.data_ptr(),
                               n_in, Fp, z.data_ptr(), z.stride(0), m.data_ptr(), win.data_ptr(),
                               torch.cuda.current_stream().cuda_stream), "bns_sage_max_f32")
    return m, win


def _case(Fp, seed=11):
    case = _crafted(1, seed)
    assert (case.ip_in[R_LONG + 1] - case.ip_in[R_LONG]) > 256
    long_row = case.ix_in[case.ip_in[R_LONG]:case.ip_in[R_LONG + 1]]
    assert long_row.unique().numel() < long_row.numel()          # multi-edges
    nnz_in = case.ix_in.numel()
    pos = torch.cat([case.pos_in, nnz_in + case.pos_out])
    return case, pos, _y(case.n_u, Fp, seed + Fp)


@pytest.mark.parametrize("Fp", WIDTHS)
def test_forward_is_exact_and_backward_matches_float64(built, Fp):
    from bns_gcn_b200.graph import SageMax
    case, pos, y = _case(Fp)
    m, win = _forward(case.g, y.to(DEV))
    m_ref, win_ref = sage_max_reference(torch.relu(y), case.u, case.v, pos, N_IN)
    assert torch.equal(m.cpu().double(), m_ref)
    assert torch.equal(win.cpu().long(), win_ref)
    assert torch.all(m[R_EMPTY] == 0) and torch.all(win[R_EMPTY] == -1)
    assert torch.all(m.cpu()[:, :Fp:7] == 0)
    # equal nonzero values from different sources: the first in walk order won
    zk = torch.relu(y)[case.u]
    ties = (zk == m_ref[case.v]) & (zk > 0)
    assert int(torch.bincount(case.v[ties.any(1)]).max()) > 1
    yd = y.to(DEV).requires_grad_(True)
    out = SageMax.apply(yd, case.g)
    assert torch.equal(out, m)
    dm = torch.randn(N_IN, Fp, generator=torch.Generator().manual_seed(Fp))
    out.backward(dm.to(DEV))
    want = sage_max_backward_reference(y, dm, case.u, case.v, N_IN)
    got = yd.grad.cpu().double()
    assert ((got - want).norm() / want.norm()).item() < 1e-6
    assert torch.all(got[torch.relu(y) == 0] == 0)


def test_a_duplicated_source_is_credited_once(built):
    """Row 0 takes source 1 three times and source 2 once, all equal: the first entry wins, and source 1's gradient is
    d m once (a source id as the winner would credit it three times)."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import PartitionGraph, SageMax
    ip = torch.tensor([0, 4, 5, 5, 7])
    ix = torch.tensor([1, 2, 1, 1, 1, 3, 3], dtype=torch.int32)
    g = PartitionGraph(4, 0, ops.DeviceGraph.from_csr(ip.to(DEV), ix.to(DEV), 4), None, DEV)
    y = torch.tensor([[0., 0., 0., 0.], [2., 1., 0., -1.], [2., 1., 0., -1.], [5., 5., 5., 5.]], device=DEV)
    yd = y.clone().requires_grad_(True)
    SageMax.apply(yd, g).backward(torch.ones(4, 4, device=DEV))
    assert yd.grad.tolist() == [[0.] * 4, [2., 2., 0., 0.], [0.] * 4, [1.] * 4]


def test_kernels_repeat_bit_identically(built):
    from bns_gcn_b200.graph import SageMax
    case, _, y = _case(604, seed=5)
    dm = torch.randn(N_IN, 604, generator=torch.Generator().manual_seed(1)).to(DEV)
    runs = []
    for _ in range(2):
        yd = y.to(DEV).requires_grad_(True)
        out = SageMax.apply(yd, case.g)
        out.backward(dm)
        runs.append((out.detach().clone(), _forward(case.g, y.to(DEV))[1], yd.grad.clone()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def _full(case):
    """The inner matrix as a homogeneous graph (square: every column is a row)."""
    from bns_gcn_b200 import ops
    return ops.DeviceGraph.from_csr(case.ip_in.to(DEV), case.ix_in.int().to(DEV), N_IN)


@pytest.mark.parametrize("Fp", WIDTHS)
def test_infer_and_its_blocks_equal_the_reference_bit_for_bit(built, Fp):
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import sage_max_infer, sage_max_infer_block
    case, _, y = _case(Fp, seed=7)
    z = torch.relu(y[:N_IN]).contiguous()
    z[3] = -0.0                                             # -0 and +0 tie: stored as +0 whatever the order
    a = _full(case)
    single = sage_max_infer(a, z.to(DEV))
    rows = torch.repeat_interleave(torch.arange(N_IN), case.ip_in[1:] - case.ip_in[:-1])
    m_ref, _ = sage_max_reference(z, case.ix_in, rows, torch.arange(case.ix_in.numel()), N_IN)
    assert torch.equal(single.cpu().double(), m_ref)
    assert not torch.signbit(single).any()
    gen = torch.Generator().manual_seed(Fp)
    for k in (1, 2, 3, 5):
        block_of = torch.randint(0, k, (N_IN,), generator=gen)
        if k > 2:
            block_of[block_of == k - 1] = 0                 # one block without entries
        order = torch.randperm(k, generator=gen).tolist()
        m = torch.empty(N_IN, Fp, device=DEV)
        seen = torch.empty(N_IN, dtype=torch.int32, device=DEV)
        for i, b in enumerate(order):
            cols = torch.nonzero(block_of == b).squeeze(1)
            renum = torch.full((N_IN,), -1, dtype=torch.int64)
            renum[cols] = torch.arange(cols.numel())
            keep = renum[case.ix_in] >= 0
            ipb = torch.zeros(N_IN + 1, dtype=torch.int64)
            ipb[1:] = torch.cumsum(torch.bincount(rows[keep], minlength=N_IN), 0)
            blk = ops.DeviceGraph.from_csr(ipb.to(DEV), renum[case.ix_in[keep]].int().to(DEV), max(cols.numel(), 1))
            zb = z[cols] if cols.numel() else torch.zeros(1, Fp)
            sage_max_infer_block(blk, zb.contiguous().to(DEV) if blk.nnz else None, m, seen, i == 0, i == k - 1, m)
        assert torch.equal(m, single), (Fp, k)


def test_malformed_arguments_are_refused(built):
    from bns_gcn_b200._lib import BnsError, lib
    from bns_gcn_b200.graph import SageMax, sage_max_infer, sage_max_infer_block
    case, _, y = _case(44, seed=3)
    a = _full(case)
    z = torch.relu(y[:N_IN]).contiguous().to(DEV)
    for bad in (z[:, :42], torch.zeros(N_IN, 1028, device=DEV), z.double(), z.cpu(), z[:-1], z[:, 4:].contiguous()[:, :36]
                .t().contiguous().t()):
        with pytest.raises(BnsError):
            sage_max_infer(a, bad)
    m = torch.empty(N_IN, 44, device=DEV)
    seen = torch.empty(N_IN, dtype=torch.int32, device=DEV)
    with pytest.raises(BnsError, match="needs z"):
        sage_max_infer_block(a, None, m, seen, True, True, m)
    with pytest.raises(BnsError, match="needs out"):
        sage_max_infer_block(a, z, m, seen, True, True, None)
    with pytest.raises(BnsError):
        sage_max_infer_block(a, z, m, seen.long(), True, True, m)
    with pytest.raises(BnsError):
        SageMax.apply(y[:, :42].contiguous().to(DEV), case.g)              # width not a multiple of 4
    st = torch.cuda.current_stream().cuda_stream
    out = torch.empty(N_IN, 44, device=DEV)
    assert lib.bns_sage_max_infer_f32(a._h, 44, None, 44, out.data_ptr(), st) != 0            # NULL z
    assert lib.bns_sage_max_infer_f32(a._h, 1032, z.data_ptr(), 1032, out.data_ptr(), st) != 0  # above 1024
    assert lib.bns_sage_max_infer_f32(a._h, 44, z.data_ptr() + 4, 44, out.data_ptr(), st) != 0  # misaligned
    assert lib.bns_sage_max_f32(None, None, None, None, None, 0, 44, z.data_ptr(), 44, out.data_ptr(), out.data_ptr(),
                                st) != 0                                                       # NULL graph
    assert lib.bns_sage_max_bwd_f32(a._h, 0, None, 0, 44, None, None, z.data_ptr(), 44, out.data_ptr(), st) != 0  # no perm
    assert lib.bns_sage_max_bwd_f32(case.g.a_in_t._h, 2 ** 31 - 10, None, 0, 44, out.data_ptr(), out.data_ptr(),
                                    z.data_ptr(), 44, out.data_ptr(), st) != 0                  # positions overflow
