"""A suspended session (`SessionState` with its `KvImage`) survives torch.save / torch.load with the default
(weights-only) loader, field for field and byte for byte."""
import io

import torch


def test_session_state_round_trips_through_torch_save():
    from videollm_online_b200.engine import KvImage
    from videollm_online_b200.inference import SessionState
    g = torch.Generator().manual_seed(0)
    img = KvImage(torch.randint(0, 256, (2 * 2 * 2 * 64 * 128 * 2,), dtype=torch.uint8, generator=g), 40, (2, 2, 128, 64))
    frames = [(3.5, torch.randn(10, 256, generator=g).to(torch.bfloat16)), (4.0, torch.randn(10, 256, generator=g).to(torch.bfloat16))]
    st = SessionState(kv=img, last_ids=torch.tensor([[11]]), video_time=4.0, last_frame_idx=8,
                      query_queue=[(3.75, "what now?")], frame_embeds_queue=frames, drafter_ids=[5, -1, -1, 7],
                      n_calls=12, started=True)
    buf = io.BytesIO()
    torch.save(st, buf)
    buf.seek(0)
    got = torch.load(buf)
    assert isinstance(got, SessionState) and isinstance(got.kv, KvImage)
    assert got.kv.n_tokens == 40 and got.kv.layout == (2, 2, 128, 64) and got.kv.event is None
    assert torch.equal(got.kv.data, img.data)
    assert torch.equal(got.last_ids, st.last_ids)
    assert (got.video_time, got.last_frame_idx, got.query_queue, got.drafter_ids, got.n_calls, got.started) == \
        (4.0, 8, [(3.75, "what now?")], [5, -1, -1, 7], 12, True)
    assert [t for t, _ in got.frame_embeds_queue] == [3.5, 4.0]
    assert all(torch.equal(a[1], b[1]) and a[1].dtype == torch.bfloat16 for a, b in zip(got.frame_embeds_queue, frames))
