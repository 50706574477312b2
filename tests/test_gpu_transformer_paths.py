"""One transformer for one pair and for a batch: ``GeometricTransformer.forward`` of one pair is ``forward_stacked`` of its two clouds
(output and gradient bits), and ``forward_train`` of one pair trains exactly as ``forward_train_batch`` of a batch of that one pair
(every parameter gradient's bits)."""
import pytest
import torch

from geotransformer_b200.loss import OverallLoss
from oracle import backbone_grad_oracle as BV

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _fresh(cfg, sd):
    from geotransformer_b200.model import create_model
    model = create_model(cfg)
    model.load_state_dict(sd, strict=True)
    return model.cuda()


def _cuda_data(data):
    return {k: ([x.cuda() if isinstance(x, torch.Tensor) else x for x in v] if isinstance(v, list) else
                (v.cuda() if isinstance(v, torch.Tensor) else v)) for k, v in data.items()}


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_pair_forward_equals_the_stacked_forward(workload, cfg_name, models):
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    dc = _cuda_data(BV.collate(workload, cfg))
    with torch.no_grad():
        feats_c = model.backbone(dc['features'], dc)[-1]
    pts = dc['points'][-1]
    n0 = int(dc['lengths'][-1][0])
    n1 = pts.shape[0] - n0
    tr = model.transformer
    ups = [u.cuda() for u in BV.upstream([(n0, cfg.geotransformer.output_dim), (n1, cfg.geotransformer.output_dim)])]

    def backward(y0, y1):
        tr.zero_grad(set_to_none=True)
        ((y0 * ups[0]).sum() + (y1 * ups[1]).sum()).backward()
        return {k: p.grad.clone() for k, p in tr.named_parameters()}

    rf, sf = feats_c[:n0].clone().requires_grad_(True), feats_c[n0:].clone().requires_grad_(True)
    y0, y1 = tr(pts[:n0].contiguous(), pts[n0:].contiguous(), rf, sf)
    want = dict(backward(y0, y1), feats=torch.cat([rf.grad, sf.grad]))
    fc = feats_c.clone().requires_grad_(True)
    y = tr.forward_stacked(pts, fc, [n0, n1])
    assert torch.equal(_bits(y), _bits(torch.cat([y0, y1])))
    got = dict(backward(y[:n0], y[n0:]), feats=fc.grad)
    assert len(got) == len(list(tr.parameters())) + 1
    for k, g in got.items():
        assert torch.equal(_bits(g), _bits(want[k])), k


@pytest.mark.parametrize('workload,cfg_name', BV.WORKLOADS)
def test_one_pair_trains_as_a_batch_of_one(workload, cfg_name, models):
    cfg, sd, _ = models(cfg_name)
    model = _fresh(cfg, sd)
    dc = _cuda_data(BV.collate(workload, cfg))
    loss = OverallLoss(cfg)
    got = []
    for forward in (model.forward_train, model.forward_train_batch):
        model.zero_grad(set_to_none=True)
        loss.graph_rows(forward(dict(dc), 7351, 3), dc)[0, 0].backward()
        got.append({k: p.grad.clone() for k, p in model.named_parameters()})
    single, batch = got
    assert len(single) == len(batch) == len(list(model.parameters()))
    for k, g in single.items():
        assert torch.equal(_bits(g), _bits(batch[k])), k
