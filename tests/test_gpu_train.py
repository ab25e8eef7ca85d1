"""End-to-end training checks of the hand-written bf16 engine (VERDICT round 1, weak #8):

(a) three epochs of the tcgen05 engine (production path: CUDA-graph replay + the four-stream slot pipeline) against
    plain fp32 PyTorch on the same synthetic shard, same initial weights, same batch order;
(b) the production path against the eager (kernel-by-kernel, no graph, no pipeline) path of the same engine over
    eight steps.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _setup(backend, dtype, use_graph, n_img=256, seed=5):
    from hefl_b200.config import FLConfig
    from hefl_b200.fl.data import BatchFeeder, SyntheticImageDataset
    from hefl_b200.fl.trainer import LocalTrainer
    from hefl_b200.models import ParamPack, create_model

    dev = torch.device("cuda")
    torch.manual_seed(seed)
    cfg = FLConfig(model="medcnn", batch_size=32, nn_backend=backend, dtype=dtype, lr=1e-3)
    model = create_model("medcnn").to(dev)
    pack = ParamPack(model)
    tr = LocalTrainer(model, pack, cfg, dev, backend=backend, use_graph=use_graph, augment=False)
    ds = SyntheticImageDataset(n_img, 256, 3, 2, seed=11)
    feed = BatchFeeder(ds, range(0, n_img), 32, dev, shuffle=True, seed=3)
    return tr, pack, feed


def _layouts_follow_weights(tr):
    """After the update (the layers above layer 1 on the side stream, layer 1 in the tail), the bf16 shadow and both
    tensor-core weight layouts hold exactly the fp32 weights."""
    eng = tr.engine
    assert torch.equal(eng.shadow, tr.pack.trainable().to(torch.bfloat16))
    Wf, Wd = torch.zeros_like(eng.Wf), torch.zeros_like(eng.Wd)
    tr.ops.conv_weight_relayout(eng.shadow, eng.table, Wf, Wd, 0, -1, eng.spack0, eng.compact0)
    assert torch.equal(eng.Wf, Wf) and torch.equal(eng.Wd, Wd)


def test_three_epochs_of_the_bf16_engine_track_fp32_pytorch():
    eng, pack_e, feed_e = _setup("tcgen05", "bf16", True)
    ref, pack_r, feed_r = _setup("cudnn", "fp32", False)
    assert torch.equal(pack_e.flat, pack_r.flat)                      # same initial weights
    h_e = eng.fit(feed_e, None, 3, early_stopping=None, reduce_lr_patience=None)
    h_r = ref.fit(feed_r, None, 3, early_stopping=None, reduce_lr_patience=None)
    print("engine :", [(round(s.loss, 4), round(s.accuracy, 3)) for s in h_e])
    print("fp32   :", [(round(s.loss, 4), round(s.accuracy, 3)) for s in h_r])
    assert h_r[-1].loss < h_r[0].loss                                 # the task is learnable, both improve
    assert h_e[-1].loss < h_e[0].loss
    assert abs(h_e[-1].loss - h_r[-1].loss) <= max(0.05 * h_r[-1].loss, 0.02)
    assert abs(h_e[-1].accuracy - h_r[-1].accuracy) <= 0.02
    # the first epoch is still in the smooth regime: the two must agree closely there. (Mid-training losses are
    # chaotic -- two fp32 runs of this test differ by 4 % in epoch 2 because of atomics ordering alone.)
    assert abs(h_e[0].loss - h_r[0].loss) <= 0.05 * h_r[0].loss
    # epoch-1 accuracy is NOT compared tightly: at loss 0.65 the logits sit at the decision boundary and the running
    # accuracy is a thresholded quantity (observed 0.512 vs 0.512 on one box, 0.574 vs 0.512 on another, with the
    # losses 0.6457 / 0.6497 both times); it only has to be in the same regime
    assert abs(h_e[0].accuracy - h_r[0].accuracy) <= 0.15
    # measured on the GPU: losses (0.6454, 0.1647, 0.0000) vs fp32 (0.6498, 0.1791, 0.0000), accuracy 1.0 / 1.0 from
    # epoch 2 on both; the trained weights stay close (bf16 activations, fp32 master weights and moments): cosine 0.9963
    cos = torch.nn.functional.cosine_similarity(pack_e.flat, pack_r.flat, dim=0).item()
    assert cos > 0.99


def test_graph_and_pipeline_path_equals_the_eager_path_over_eight_steps():
    a, pack_a, feed_a = _setup("tcgen05", "bf16", True)
    b, pack_b, feed_b = _setup("tcgen05", "bf16", False)
    a.fit(feed_a, None, 1, early_stopping=None, reduce_lr_patience=None)      # 8 steps of 32
    b.fit(feed_b, None, 1, early_stopping=None, reduce_lr_patience=None)
    torch.cuda.synchronize()
    assert int(a.step_t.item()) == int(b.step_t.item()) == 8
    _layouts_follow_weights(a)
    _layouts_follow_weights(b)
    # same kernels, same order of operations; only the fp32 atomics of the weight gradients reorder. Adam moves
    # every weight by ~lr per step whatever the size of its gradient, so a weight whose gradient is pure rounding
    # noise may drift by up to steps * lr = 8e-3 in EACH run, in opposite directions in the worst case (observed
    # maxima over boxes: 6.9e-3 ... 8.3e-3); the bulk must agree far better than that.
    d = (pack_a.flat - pack_b.flat).abs()
    print("graph vs eager: max", float(d.max()), "mean", float(d.mean()),
          "share above 4e-3:", float((d > 4e-3).float().mean()))
    assert float(d.max()) <= 2 * 8 * 1e-3
    assert float(d.mean()) < 6e-4
    assert torch.nn.functional.cosine_similarity(pack_a.flat, pack_b.flat, dim=0).item() > 0.9995
