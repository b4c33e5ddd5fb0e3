"""-m gpu: the recapture rule of captured steps.  A captured graph holds raw pointers into the encoder / decoder scratch
buffers; once a larger batch reallocates one, the graph of predict_batch_graphed and every BatchStream slot report stale
and are captured again before their next replay.  The staleness is asserted before anything is replayed, so a wrong
check fails an assertion instead of replaying a graph with stale pointers."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_scratch_growth_recaptures_before_replay(cuda_device):
    from dad_3dheads_b200.encoder_weights import synthetic_state_dict
    from dad_3dheads_b200.predictor import FaceMeshPredictor
    pred = FaceMeshPredictor.dad_3dnet(state_dict=synthetic_state_dict(0), precision="fp16x2", cuda_id=cuda_device.index or 0)
    g = torch.Generator().manual_seed(5)
    x = torch.randint(0, 256, (2, 256, 256, 3), dtype=torch.uint8, generator=g)
    keys = ("3dmm_params", "points", "3d_vertices", "landmarks_445")

    pred.predict_batch_graphed(x)
    (step,) = pred._graphs.values()
    graph = step.graph
    st = pred.open_stream(tuple(x.shape), keys=keys, depth=2)
    slot_graphs = [s["step"].graph for s in st.slots]
    assert not step.stale() and not any(s["step"].stale() for s in st.slots)

    generation = pred._ws_generation()
    big = torch.randint(0, 256, (64, 256, 256, 3), dtype=torch.uint8, generator=g)
    pred.predict_batch(big.to(cuda_device))
    torch.cuda.synchronize()
    assert pred._ws_generation() != generation
    assert step.stale()
    assert all(s["step"].stale() for s in st.slots)

    eager = {k: v.clone() for k, v in pred.predict_batch(x.to(cuda_device)).items()}
    got = pred.predict_batch_graphed(x)
    assert list(pred._graphs.values()) == [step] and step.graph is not graph and not step.stale()
    assert got.keys() == eager.keys()
    for k in eager:
        assert torch.equal(got[k], eager[k]), k

    st.submit(x.pin_memory())
    res = st.collect()
    assert st.slots[0]["step"].graph is not slot_graphs[0] and not st.slots[0]["step"].stale()
    assert st.slots[0]["out"] is st.slots[0]["step"].out
    assert st.slots[1]["step"].stale()                          # not submitted to since the growth: not replayed
    for k in keys:
        assert torch.equal(res[k], eager[k].cpu()), k
