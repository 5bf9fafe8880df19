"""GpuContext.close() closes the models still open on it first: snnb_model_destroy uses the model's context, so a model that outlives
its context (kept alive by a reference cycle, say, and collected after the context was closed) must have nothing left to destroy."""
import pytest

from shadernn_b200 import core, modelzoo

pytestmark = pytest.mark.gpu


def test_closing_a_context_closes_its_open_models(built, tmp_path):
    b = modelzoo.Builder(seed=7)
    b.conv(b.input(16, 8, 1), 1, 3)
    path = modelzoo.write_model(b.layers, str(tmp_path / "tiny.json"))
    ctx = core.GpuContext(0)
    kept, closed = core.MixedInferenceCore(ctx, path), core.MixedInferenceCore(ctx, path)
    closed.close()
    assert kept.h and not closed.h
    ctx.close()
    assert not ctx.h and not kept.h, "the context was destroyed under an open model"
    kept.close()  # nothing left to do
    closed.close()
