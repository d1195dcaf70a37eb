"""One chunk of the Qwen3-ASR realtime model for N streams, with the frame rows kept where the engines run.

The reference's ``append_audio_to_cache`` (third_party/qwen3-asr-causal/src/qwen3_asr_causal/model.py:809-836 and, with a
mutable tail, causal.py:823-864) runs tower -> frame adapter -> ``torch.cat`` onto ``state.frame_hidden`` per stream.
``RealtimeFrames.append`` does the same for N streams at once:

  1. the tower for every stream in one engine call (``B200QwenAudioCausalKVEncoder.encode_rows``);
  2. one ``adapt`` of the text engine over all new rows (``wlk_qtext_adapt`` on the device);
  3. each stream's rows written into its own frame buffer, an fp32 tensor grown geometrically, so that
     ``state.frame_hidden`` is a ``[1, steps, d]`` view of it: append-only, or the mutable tail replaced in place.

``B200QwenTextDecoder.generate_rolling_batch`` then runs ``generate_full_hypothesis_rolling`` for the N streams in one
lockstep pass of the text driver, which forwards only each stream's delta rows.  With device engines no frame row
reaches the host; with the CPU oracles behind the same engine API the buffers are CPU tensors and the same code runs."""
from __future__ import annotations

from typing import Optional, Sequence

_MIN_CAP = 64


def _own_prefix(fh, buf) -> bool:
    """Whether the view fh [1, steps, d] is the first `steps` rows of buf [cap, d]."""
    if fh.shape[1] == 0:
        return True
    return (buf is not None and fh.device == buf.device and fh.shape[1] <= buf.shape[0] and fh.data_ptr() == buf.data_ptr()
            and fh.stride(1) == buf.stride(0) and fh.stride(2) == 1)


class RealtimeFrames:
    """The frame half of the realtime model for N streams over one tower encoder and one text engine."""

    def __init__(self, encoder, text_engine, d_model: int):
        self.encoder, self.text, self.d = encoder, text_engine, int(d_model)

    def _buffer(self, state, steps_needed: int, device):
        """The stream's buffer, holding state.frame_hidden as its prefix and room for steps_needed rows.  A view the
        caller put in state.frame_hidden that is not such a prefix (the streamer's [:, -k:] trim at rollover) is copied
        into a fresh buffer."""
        import torch
        buf = getattr(state, "_b200_frames", None)
        fh = state.frame_hidden
        steps = 0 if fh is None else int(fh.shape[1])
        if fh is not None and not _own_prefix(fh, buf):
            src = fh[0]
            buf = None
        else:
            src = None
        if buf is None or buf.shape[0] < steps_needed:
            cap = max(_MIN_CAP, steps_needed, steps, 2 * (0 if buf is None else buf.shape[0]))
            new = torch.empty(cap, self.d, dtype=torch.float32, device=device)
            if steps:
                new[:steps].copy_(src if src is not None else buf[:steps])
            buf = new
            state._b200_frames = buf
        return buf

    def append(self, states: Sequence, mels: Optional[Sequence] = None, flush: bool = False):
        """append_audio_to_cache (flush=False) or flush_audio_to_cache (flush=True) for N CachedAudioDecodeStates.
        Returns (cached, delta) per stream, both [1, steps, d] views."""
        import torch
        audio = [st.audio for st in states]
        previous_mutable = [int(getattr(a, "mutable_steps", 0)) for a in audio]
        mutable = self.encoder.mutable_tail_steps > 0 and not flush
        rows, offs = self.encoder.encode_rows(audio, mels, flush=flush)
        adapted = self.text.adapt(rows) if rows.shape[0] else rows.new_zeros(0, self.d)
        out = []
        for i, st in enumerate(states):
            new = adapted[offs[i]: offs[i + 1]]
            n = int(new.shape[0])
            steps = 0 if st.frame_hidden is None else int(st.frame_hidden.shape[1])
            if mutable:                                     # causal.py:850-864: the previous tail is replaced
                at = steps - previous_mutable[i]
                if at < 0:
                    raise ValueError("cached frame_hidden shorter than the previous mutable tail")
            else:
                at = steps
            buf = self._buffer(st, at + n, adapted.device)
            if n:
                buf[at: at + n].copy_(new)
            st.frame_hidden = buf[None, : at + n]
            if mutable:
                st.adapter.audio_frames_seen += int(mels[i].shape[1])
                st.adapter.decoder_steps_seen = at + n
                delta = buf[None, at + previous_mutable[i]: at + n]
            else:                                           # adapter.forward_chunk's counters (model.py:676-683)
                st.adapter.audio_frames_seen += n
                st.adapter.decoder_steps_seen += n
                delta = buf[None, at: at + n]
            out.append((st.frame_hidden, delta))
        if rows.is_cuda:
            torch.cuda.current_stream(rows.device).synchronize()
        return out

