"""The next step's front-end starts behind the backward-data pass (tcr_step_args::input_resident), so at full batch it runs beside
the weight-gradient launch, which still reads the current step's features.  Running ahead must not change a bit: same inputs and
seeds, ordered against ahead, over both feature buffers, at the batch sizes where the two launches overlap most."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("model,width,n", [("TCResNet8", 1.0, 512), ("TCResNet14", 1.5, 1024)])
def test_frontend_ahead_of_weight_gradients_is_bitwise_equal(model, width, n):
    import torch
    from tcresnet_b200.engine import Engine
    gen = torch.Generator(device="cuda").manual_seed(5)
    wavs = [torch.rand(n, 16000, device="cuda", generator=gen) * 2 - 1 for _ in range(3)]
    hots = [torch.nn.functional.one_hot(torch.randint(0, 12, (n,), device="cuda", generator=gen), 12).float() for _ in range(3)]
    results = []
    for ahead in (False, True):
        eng = Engine(model=model, width_multiplier=width, max_batch=n, dropout_keep_prob=0.5)
        p, s, m = eng.new_variables(seed=0)
        losses = []
        for i in range(6):
            out = eng.train_step(wavs[i % 3], hots[i % 3], p, s, m, 0.05, dropout_seed=i, want_grads=True, input_resident=ahead)
            losses.append(out["losses"].clone())
        torch.cuda.synchronize()
        results.append((p.clone(), s.clone(), m.clone(), out["grads"].clone(), torch.stack(losses)))
        eng.close()
    for x, y in zip(*results):
        assert torch.equal(x, y)
