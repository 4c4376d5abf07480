"""Host side of the per-item text windows of the FLUX joint attention: mask validation, window construction for left and
right padding, and stack_prompt_embeds.  No GPU needed."""
import pytest
import torch

from gpt_image_edit_b200._lib import B2FError
from gpt_image_edit_b200.flux_transformer import text_windows
from gpt_image_edit_b200.pipeline import stack_prompt_embeds


def test_windows_of_left_and_right_padding():
    m = torch.tensor([[0, 0, 1, 1, 1],     # left-padded (Qwen processor), then T5: the run ends at S_txt
                      [1, 1, 1, 1, 1],     # unpadded: the full window
                      [1, 1, 0, 0, 0],     # right-padded
                      [0, 1, 1, 0, 0],     # padded on both sides: still one run
                      [0, 0, 0, 0, 1]])
    w = text_windows(m, 5, 5)
    assert w.dtype == torch.int32 and w.device.type == "cpu"
    assert w.tolist() == [[2, 5], [0, 5], [0, 2], [1, 3], [4, 5]]
    assert text_windows(m.bool(), 5, 5).tolist() == w.tolist()


@pytest.mark.parametrize("row", [[1, 0, 1, 1], [0, 1, 0, 1], [1, 1, 0, 1]])
def test_rows_with_holes_are_refused(row):
    with pytest.raises(B2FError, match="contiguous"):
        text_windows(torch.tensor([[1, 1, 1, 1], row]), 2, 4)


def test_empty_rows_are_refused():
    with pytest.raises(B2FError, match="empty"):
        text_windows(torch.tensor([[1, 1, 1], [0, 0, 0]]), 2, 3)


@pytest.mark.parametrize("shape", [(2, 4), (3, 5), (3,), (3, 4, 1)])
def test_shape_mismatches_are_refused(shape):
    with pytest.raises(B2FError, match="expected"):
        text_windows(torch.ones(shape, dtype=torch.int64), 3, 4)


def test_stack_prompt_embeds_left_pads_like_the_processor():
    g = torch.Generator().manual_seed(0)
    lens = [5, 2, 7]
    embeds = [torch.randn(1, n, 8, generator=g).bfloat16() for n in lens]
    e, m = stack_prompt_embeds(embeds)
    assert e.shape == (3, 7, 8) and e.dtype == torch.bfloat16
    assert m.shape == (3, 7) and m.dtype == torch.int64
    for b, n in enumerate(lens):
        assert torch.equal(e[b, 7 - n:], embeds[b][0])
        assert not e[b, :7 - n].any()
        assert m[b].tolist() == [0] * (7 - n) + [1] * n
    assert text_windows(m, 3, 7).tolist() == [[2, 7], [5, 7], [0, 7]]


def test_stack_prompt_embeds_refusals():
    with pytest.raises(ValueError):
        stack_prompt_embeds([])
    with pytest.raises(ValueError):
        stack_prompt_embeds([torch.zeros(1, 3, 8), torch.zeros(1, 3, 4)])    # widths differ
    with pytest.raises(ValueError):
        stack_prompt_embeds([torch.zeros(2, 3, 8)])                          # not one prompt
    with pytest.raises(ValueError):
        stack_prompt_embeds([torch.zeros(1, 0, 8)])                          # empty prompt
