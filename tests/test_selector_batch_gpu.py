"""The batched viewpoint selection against itself one query at a time: Q queries through one call give, query for query,
the logits, angles and S2 scores of Q calls of one query, bit for bit (torch.equal), at bench.py's shapes (64 references
x 5 angles, 10 crops) and for two reference records selected against in turn, one of them over more queries than a
chunk holds."""
import pytest
import torch

from golden import cases
from gen6d_b200 import ops
from gen6d_b200.network import name2network
from gen6d_b200.network.selector import SEL_QUERY_CHUNK
from gen6d_b200.weights import seeded_state_dict

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def net():
    c = cases.selector_case(rfn=64, an=5, qn=1)
    net = name2network['selector'](c['cfg'])
    net.load_state_dict(seeded_state_dict(net, cases.WEIGHT_SEED), strict=True)
    net.cuda().eval()
    return net


def query_feats(net, seed, qn):
    c = cases.selector_case(seed=seed, rfn=1, an=1, qn=qn)
    x = ops.preprocess_u8(torch.from_numpy(c['que_imgs']).cuda(), out_c=4, imagenet_norm=True)
    return net._feats(x)


def assert_batch_is_per_query(net, feats, refs=None, counters=None):
    qn = feats[0].shape[0]
    with torch.no_grad():
        got = net._select_batch(feats, refs, counters)
        one = [net._select_batch([f[q:q + 1] for f in feats], refs, counters) for q in range(qn)]
    torch.cuda.synchronize()
    for name, g, parts in zip(('logits', 'angles', 'scores'), got, zip(*one)):
        want = torch.cat(parts, 0)
        assert g.shape == want.shape, name
        assert torch.equal(g, want), (name, (g - want).abs().max().item())
    return got


def test_batched_selection_is_per_query_at_bench_shapes(net):
    c = cases.selector_case(rfn=64, an=5, qn=1)
    net.load_ref_imgs(c['ref_imgs'], c['ref_poses'], c['object_center'], c['object_vert'])
    logits, angles, scores = assert_batch_is_per_query(net, query_feats(net, 3, 10))
    assert logits.shape == (10, 64) and angles.shape == (10, 64) and scores.shape == (10, 3, 320)
    assert torch.isfinite(logits).all() and torch.isfinite(angles).all()


def test_batched_selection_is_per_query_for_two_records(net):
    """Two reference records, each with its own S2 counters, as an object set selects against them slot by slot; the
    second over more queries than one chunk holds."""
    recs = []
    for seed in (41, 53):
        c = cases.selector_case(seed=seed, rfn=64, an=5, qn=1)
        refs = net.make_refs(c['ref_imgs'], c['ref_poses'], c['object_center'], c['object_vert'])
        recs.append((refs, net.s2_counters_for(refs, net.device)))
    for (refs, counters), qn in zip(recs, (4, SEL_QUERY_CHUNK + 2)):
        assert_batch_is_per_query(net, query_feats(net, 7 + qn, qn), refs, counters)
    with pytest.raises(ValueError):
        net._select_batch(query_feats(net, 5, 1), recs[0][0], None)
