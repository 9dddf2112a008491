"""GPU: the single-sequence fused decode step's self-validating exchange words alternate between two sets, selected by
the parity of that kernel's own count of executed launches.  The batched kernel shares the launch epoch but not that
count, so interleaving the two kernels on one session must leave every set clean for the launch that uses it."""
import pytest

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth


@pytest.mark.gpu
def test_exchange_sets_alternate_across_interleaved_kernels(tiny):
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, model = tiny
    one_odd = [synth.make_clip(70, 4.0)]
    five = [synth.make_clip(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1])]
    one_even = [synth.make_clip(71, 12.3)]
    runs = [  # (clips, batched kernel, max_new_tokens)
        (one_odd, "0", 13),      # single-sequence kernel, 12 launches
        (five, "0", 10),         # single-sequence kernel, 5 launches per step
        (five, "1", 14),         # batched kernel: 13 steps, an odd number of launch epochs
        (one_even, "0", 12),     # single-sequence kernel again
    ]
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    try:
        # one session for all four runs (the engine re-creates it when a batch outgrows it): exchange words and counters
        # carry over from run to run
        longest = max(c.shape[0] for clips, _, _ in runs for c in clips)
        eng._ensure_session(5, longest, 0, max(n for _, _, n in runs))
        for clips, batch_step, n_new in runs:
            eng.set_option("batch_step", batch_step)
            before = eng.stats()
            got = eng.transcribe_ids(clips, max_new_tokens=n_new)
            after = eng.stats()
            kernel = "decode_batch_steps" if batch_step == "1" else "decode_fused_steps"
            assert after[kernel] - before[kernel] == n_new - 1, (batch_step, n_new)
            assert after["decode_phase_steps"] == before["decode_phase_steps"]
            for g, c in zip(got.ids, clips):
                assert g == O.transcribe_ids(model, c, max_new_tokens=n_new).ids, (batch_step, n_new)
    finally:
        eng.close()
