//! Safe wrapper over `ffi.rs`: RAII handles in the style of `MlxArray` (`src/backend/mlx/array.rs:15-29`),
//! status codes turned into `anyhow::Error` (the reference's module-level error type, `src/inference.rs:30,89`).
//! No `Tensor` crosses this boundary: the hot span of `transcribe()` (steps 2-8, `src/inference.rs:94-200`) is one call.
pub mod ffi;

use anyhow::{anyhow, Result};
use std::ffi::{CStr, CString};
use std::ptr;

fn check(status: i32) -> Result<()> {
    if status == ffi::ASRB_OK { return Ok(()); }
    let msg = unsafe { CStr::from_ptr(ffi::asrb_last_error()) }.to_string_lossy().into_owned();
    Err(anyhow!("asr_b200 error {status}: {msg}"))
}

struct Ctx(*mut ffi::asrb_ctx);
impl Drop for Ctx { fn drop(&mut self) { unsafe { ffi::asrb_ctx_free(self.0); } } }
struct Model(*mut ffi::asrb_model);
impl Drop for Model { fn drop(&mut self) { unsafe { ffi::asrb_model_free(self.0); } } }
struct Session(*mut ffi::asrb_session);
impl Drop for Session { fn drop(&mut self) { unsafe { ffi::asrb_session_free(self.0); } } }

/// Device context + immutable weights + one session (KV cache, scratch, stream) for batch-1 `transcribe()` calls.
/// The session is created lazily and re-created only when a clip is longer than its capacity (the reference handles
/// arbitrary-length audio; a session sized for the worst case up front would pin ~1 GB of scratch per minute of audio).
/// Field order = drop order: session before model before context.
pub struct B200Engine {
    session: std::cell::RefCell<Option<(Session, usize, usize, usize)>>,   // (handle, capacity in samples, slots, context ids)
    model: Model,
    _ctx: Ctx,
    max_new_tokens: usize,
}

// `transcribe(&self)` is `&self` in the reference and single-threaded (`src/inference.rs:89`); a session is not
// re-entrant, so the engine is Send but deliberately not Sync.
unsafe impl Send for B200Engine {}

impl B200Engine {
    /// Replaces the loaders of `AsrInference::load` (`src/inference.rs:39-74`): config.json + safetensors (single or
    /// sharded) are read by the library, bf16 stays bf16.
    pub fn load(model_dir: &str, device: i32, max_new_tokens: usize) -> Result<Self> {
        let mut ctx = ptr::null_mut();
        check(unsafe { ffi::asrb_init(device, &mut ctx) })?;
        let ctx = Ctx(ctx);
        let dir = CString::new(model_dir)?;
        let mut model = ptr::null_mut();
        check(unsafe { ffi::asrb_model_load(ctx.0, dir.as_ptr(), &mut model) })?;
        let model = Model(model);
        Ok(Self { session: std::cell::RefCell::new(None), model, _ctx: ctx, max_new_tokens })
    }

    /// Session with room for `n_samples`: capacity grows in 30 s steps, the old session is dropped first.
    fn session_for(&self, n_samples: usize) -> Result<*mut ffi::asrb_session> { self.session_for_slots(n_samples, 1) }

    /// Session with room for `n_samples` and `slots` decode rows (a beam search of K needs K); neither shrinks.
    fn session_for_slots(&self, n_samples: usize, slots: usize) -> Result<*mut ffi::asrb_session> {
        self.session_for_context(n_samples, slots, 0)
    }

    /// Session with room for `n_samples`, `slots` decode rows and `n_context` context ids; none of them shrinks, and
    /// the context capacity grows in steps of 256 ids.
    fn session_for_context(&self, n_samples: usize, slots: usize, n_context: usize) -> Result<*mut ffi::asrb_session> {
        let mut slot = self.session.borrow_mut();
        let (mut rows, mut ctx_cap) = (slots, (n_context + 255) / 256 * 256);
        if let Some((s, cap, have, have_ctx)) = slot.as_ref() {
            if *cap >= n_samples && *have >= slots && *have_ctx >= n_context { return Ok(s.0); }
            rows = rows.max(*have);
            ctx_cap = ctx_cap.max(*have_ctx);
        }
        *slot = None;
        let cap = ((n_samples + 479_999) / 480_000).max(1) * 480_000;
        let mut session = ptr::null_mut();
        check(unsafe {
            ffi::asrb_session_create_ex(self.model.0, rows as i32, cap as i64, 16, ctx_cap as i32, self.max_new_tokens as i32,
                                        &mut session)
        })?;
        *slot = Some((Session(session), cap, rows, ctx_cap));
        Ok(session)
    }

    pub fn dims(&self) -> Result<ffi::AsrbDims> {
        let mut d = ffi::AsrbDims::default();
        check(unsafe { ffi::asrb_model_dims(self.model.0, &mut d) })?;
        Ok(d)
    }

    /// Steps 2-8 of `transcribe()`: 16 kHz mono f32 samples (+ optional forced-language prompt ids,
    /// `src/inference.rs:246-250`) -> generated token ids, EOS excluded.
    pub fn transcribe_ids(&self, samples: &[f32], lang_ids: Option<&[i64]>) -> Result<Vec<i64>> {
        let mut ids = vec![0i32; self.max_new_tokens];
        let mut n = 0i32;
        let sp = [samples.as_ptr()];
        let sl = [samples.len() as i64];
        let lp = [lang_ids.map_or(ptr::null(), |v| v.as_ptr())];
        let ll = [lang_ids.map_or(0, |v| v.len() as i32)];
        let session = self.session_for(samples.len())?;
        check(unsafe {
            ffi::asrb_transcribe_ids(session, sp.as_ptr(), sl.as_ptr(), 1, lp.as_ptr(), ll.as_ptr(),
                                     self.max_new_tokens as i32, ids.as_mut_ptr(), &mut n)
        })?;
        Ok(ids[..n as usize].iter().map(|&t| t as i64).collect())
    }

    /// `transcribe_ids` that also returns the natural-log probability of every generated id and of the EOS id that
    /// ended the sequence (`None` when it stopped at `max_new_tokens`), computed by the decode kernels from the same
    /// fp32 logits that selected the ids (`asrb_last_logprobs`).  The ids are those `transcribe_ids` returns.
    pub fn transcribe_ids_with_logprobs(&self, samples: &[f32], lang_ids: Option<&[i64]>) -> Result<(Vec<i64>, Vec<f32>, Option<f32>)> {
        let session = self.session_for(samples.len())?;
        let key = CString::new("logprobs")?;
        let on = CString::new("1")?;
        let off = CString::new("0")?;
        check(unsafe { ffi::asrb_session_set_option(session, key.as_ptr(), on.as_ptr()) })?;
        let run = (|| -> Result<(Vec<i64>, Vec<f32>, Option<f32>)> {
            let ids = self.transcribe_ids(samples, lang_ids)?;
            let mut lp = vec![0f32; self.max_new_tokens];
            let mut eos = 0f32;
            check(unsafe { ffi::asrb_last_logprobs(session, self.max_new_tokens as i32, lp.as_mut_ptr(), &mut eos) })?;
            lp.truncate(ids.len());
            Ok((ids, lp, if eos.is_nan() { None } else { Some(eos) }))
        })();
        check(unsafe { ffi::asrb_session_set_option(session, key.as_ptr(), off.as_ptr()) })?;
        run
    }

    /// `transcribe_ids` that also returns, for every generated id, the `k` (1..=8) best candidates of the decode step
    /// that selected it as `(id, natural-log probability)` pairs, best first (entry 0 is the id itself), and the same
    /// for the step that selected the EOS ending the sequence (`None` when it stopped at `max_new_tokens`).  The
    /// candidates come from the decode kernels, under the same fp32 logits that selected the ids
    /// (`asrb_last_top_logprobs`).  The ids are those `transcribe_ids` returns.
    pub fn transcribe_ids_with_top_logprobs(&self, samples: &[f32], lang_ids: Option<&[i64]>, k: usize)
        -> Result<(Vec<i64>, Vec<Vec<(i64, f32)>>, Option<Vec<(i64, f32)>>)> {
        if !(1..=8).contains(&k) { return Err(anyhow!("top_logprobs k must be in 1..=8, got {k}")); }
        let session = self.session_for(samples.len())?;
        let key = CString::new("top_logprobs")?;
        let on = CString::new(k.to_string())?;
        let off = CString::new("0")?;
        check(unsafe { ffi::asrb_session_set_option(session, key.as_ptr(), on.as_ptr()) })?;
        let run = (|| -> Result<(Vec<i64>, Vec<Vec<(i64, f32)>>, Option<Vec<(i64, f32)>>)> {
            let ids = self.transcribe_ids(samples, lang_ids)?;
            let mut cid = vec![-1i32; self.max_new_tokens * k];
            let mut clp = vec![0f32; self.max_new_tokens * k];
            let mut eid = vec![-1i32; k];
            let mut elp = vec![0f32; k];
            check(unsafe {
                ffi::asrb_last_top_logprobs(session, self.max_new_tokens as i32, k as i32, cid.as_mut_ptr(), clp.as_mut_ptr(),
                                            eid.as_mut_ptr(), elp.as_mut_ptr())
            })?;
            let rows = (0..ids.len())
                .map(|t| (0..k).map(|j| (cid[t * k + j] as i64, clp[t * k + j])).collect())
                .collect();
            let eos = if eid[0] < 0 { None } else { Some((0..k).map(|j| (eid[j] as i64, elp[j])).collect()) };
            Ok((ids, rows, eos))
        })();
        check(unsafe { ffi::asrb_session_set_option(session, key.as_ptr(), off.as_ptr()) })?;
        run
    }

    /// `transcribe_ids` with seeded temperature sampling: every id is drawn by the decode kernels from
    /// softmax(logits / `temperature`) with the Gumbel-max draw of the options "temperature" / "seed"
    /// (`include/asr_b200.h`).  `temperature` 0 is greedy, else finite in [1e-6, 100]; its shortest decimal form is what
    /// the library parses.  The ids are a pure function of (samples, language prompt, seed, temperature).  The options
    /// are set for this call and restored to greedy / seed 0 afterwards.
    pub fn transcribe_ids_sampled(&self, samples: &[f32], lang_ids: Option<&[i64]>, temperature: f32, seed: u64) -> Result<Vec<i64>> {
        let session = self.session_for(samples.len())?;
        let tkey = CString::new("temperature")?;
        let skey = CString::new("seed")?;
        let tval = CString::new(format!("{temperature}"))?;
        let sval = CString::new(seed.to_string())?;
        let zero = CString::new("0")?;
        let set = (|| -> Result<()> {
            check(unsafe { ffi::asrb_session_set_option(session, tkey.as_ptr(), tval.as_ptr()) })?;
            check(unsafe { ffi::asrb_session_set_option(session, skey.as_ptr(), sval.as_ptr()) })
        })();
        let run = set.and_then(|_| self.transcribe_ids(samples, lang_ids));
        check(unsafe { ffi::asrb_session_set_option(session, tkey.as_ptr(), zero.as_ptr()) })?;
        check(unsafe { ffi::asrb_session_set_option(session, skey.as_ptr(), zero.as_ptr()) })?;
        run
    }

    /// `transcribe_ids` with the repetition controls, the options "no_repeat_ngram_size" / "repetition_penalty"
    /// (`include/asr_b200.h`): `no_repeat_ngram_size` N in 0..=16 (0: off) bans every id that would repeat an N-gram of
    /// the ids generated so far, `repetition_penalty` in [1, 10] (1: off) divides the positive and multiplies the negative
    /// logits of those ids.  The options are set for this call and restored to off afterwards.
    pub fn transcribe_ids_no_repeat(&self, samples: &[f32], lang_ids: Option<&[i64]>, no_repeat_ngram_size: u32,
                                    repetition_penalty: f64) -> Result<Vec<i64>> {
        if no_repeat_ngram_size > 16 { return Err(anyhow!("no_repeat_ngram_size must be in 0..=16, got {no_repeat_ngram_size}")); }
        if !(1.0..=10.0).contains(&repetition_penalty) {
            return Err(anyhow!("repetition_penalty must be in [1, 10], got {repetition_penalty}"));
        }
        let session = self.session_for(samples.len())?;
        let nkey = CString::new("no_repeat_ngram_size")?;
        let pkey = CString::new("repetition_penalty")?;
        let nval = CString::new(no_repeat_ngram_size.to_string())?;
        let pval = CString::new(format!("{repetition_penalty:?}"))?;
        let (zero, one) = (CString::new("0")?, CString::new("1")?);
        let set = (|| -> Result<()> {
            check(unsafe { ffi::asrb_session_set_option(session, nkey.as_ptr(), nval.as_ptr()) })?;
            check(unsafe { ffi::asrb_session_set_option(session, pkey.as_ptr(), pval.as_ptr()) })
        })();
        let run = set.and_then(|_| self.transcribe_ids(samples, lang_ids));
        check(unsafe { ffi::asrb_session_set_option(session, nkey.as_ptr(), zero.as_ptr()) })?;
        check(unsafe { ffi::asrb_session_set_option(session, pkey.as_ptr(), one.as_ptr()) })?;
        run
    }

    /// `transcribe_ids` with context biasing: `context_ids` (the tokenizer's ids of a keyword list, names or related
    /// text) become the content of the prompt's system turn (`asrb_session_set_context`).  An empty slice is the plain
    /// prompt.  The context is cleared again after the call.
    pub fn transcribe_ids_with_context(&self, samples: &[f32], lang_ids: Option<&[i64]>, context_ids: &[i64]) -> Result<Vec<i64>> {
        let session = self.session_for_context(samples.len(), 1, context_ids.len())?;
        let cp = [context_ids.as_ptr()];
        let cl = [context_ids.len() as i32];
        let run = check(unsafe { ffi::asrb_session_set_context(session, 1, cp.as_ptr(), cl.as_ptr()) })
            .and_then(|_| self.transcribe_ids(samples, lang_ids));
        check(unsafe { ffi::asrb_session_set_context(session, 0, ptr::null(), ptr::null()) })?;
        run
    }

    /// `transcribe_ids` with beam search of `beam_size` (2..=6) beams, the options "beam_size" / "length_penalty"
    /// (`include/asr_b200.h`; `length_penalty` None scores by sum / length).  Returns the `beam_size` hypotheses
    /// ranked best first as (ids, sum of log-probabilities, score, EOS id or -1 when stopped by `max_new_tokens`);
    /// entry 0 is what `transcribe_ids` would return under these options.  The options are restored afterwards.
    pub fn transcribe_ids_beam(&self, samples: &[f32], lang_ids: Option<&[i64]>, beam_size: usize, length_penalty: Option<f32>)
        -> Result<Vec<(Vec<i64>, f32, f32, i64)>> {
        if !(2..=6).contains(&beam_size) { return Err(anyhow!("beam_size must be in 2..=6, got {beam_size}")); }
        let session = self.session_for_slots(samples.len(), beam_size)?;
        let bkey = CString::new("beam_size")?;
        let lkey = CString::new("length_penalty")?;
        let bval = CString::new(beam_size.to_string())?;
        let lval = CString::new(length_penalty.map_or("none".to_string(), |a| format!("{a}")))?;
        let (one, none) = (CString::new("1")?, CString::new("none")?);
        let set = (|| -> Result<()> {
            check(unsafe { ffi::asrb_session_set_option(session, bkey.as_ptr(), bval.as_ptr()) })?;
            check(unsafe { ffi::asrb_session_set_option(session, lkey.as_ptr(), lval.as_ptr()) })
        })();
        let run = set.and_then(|_| self.transcribe_ids(samples, lang_ids)).and_then(|_| {
            let (k, m) = (beam_size, self.max_new_tokens);
            let mut ids = vec![-1i32; k * m];
            let mut lens = vec![0i32; k];
            let mut sums = vec![0f32; k];
            let mut scores = vec![0f32; k];
            let mut eos = vec![-1i32; k];
            check(unsafe {
                ffi::asrb_last_nbest(session, m as i32, k as i32, ids.as_mut_ptr(), lens.as_mut_ptr(), sums.as_mut_ptr(),
                                     scores.as_mut_ptr(), eos.as_mut_ptr())
            })?;
            Ok((0..k).map(|j| (ids[j * m..j * m + lens[j] as usize].iter().map(|&t| t as i64).collect(), sums[j], scores[j],
                               eos[j] as i64)).collect())
        });
        check(unsafe { ffi::asrb_session_set_option(session, bkey.as_ptr(), one.as_ptr()) })?;
        check(unsafe { ffi::asrb_session_set_option(session, lkey.as_ptr(), none.as_ptr()) })?;
        run
    }

    /// Word timing (`asrb_align_ids`, `include/asr_b200.h`): the start and end, in 10 ms mel frames, of every id
    /// `ids[text_from..]` in `samples`, from the decoder's attention over the audio in one teacher-forced pass over the
    /// prompt and `ids` (normally the decoded ids followed by EOS 151645).  `heads`: (layer, query head) pairs, empty =
    /// every head of the second half of the layers.  `ids.len()` may not exceed `max_new_tokens`.
    pub fn align_ids(&self, samples: &[f32], lang_ids: Option<&[i64]>, ids: &[i64], text_from: usize, heads: &[(i32, i32)])
        -> Result<Vec<(i32, i32)>> {
        if ids.is_empty() || text_from >= ids.len() { return Err(anyhow!("need text_from < ids.len() and a non-empty ids")); }
        let n = ids.len();
        let (mut st, mut en) = (vec![-1i32; n], vec![-1i32; n]);
        let sp = [samples.as_ptr()];
        let sl = [samples.len() as i64];
        let lp = [lang_ids.map_or(ptr::null(), |v| v.as_ptr())];
        let ll = [lang_ids.map_or(0, |v| v.len() as i32)];
        let ip = [ids.as_ptr()];
        let il = [n as i32];
        let tf = [text_from as i32];
        let hs: Vec<i32> = heads.iter().flat_map(|&(l, h)| [l, h]).collect();
        let session = self.session_for(samples.len())?;
        check(unsafe {
            ffi::asrb_align_ids(session, sp.as_ptr(), sl.as_ptr(), 1, lp.as_ptr(), ll.as_ptr(), ip.as_ptr(), il.as_ptr(),
                                tf.as_ptr(), if hs.is_empty() { ptr::null() } else { hs.as_ptr() }, heads.len() as i32,
                                n as i32, st.as_mut_ptr(), en.as_mut_ptr())
        })?;
        Ok((text_from..n).map(|i| (st[i], en[i])).collect())
    }

    /// One live stream on a session of its own (dropped with the returned handle): push 16 kHz mono f32 audio as it
    /// arrives and get the hypothesis of everything received so far (`asrb_stream_push`, one stream).  `max_samples`
    /// bounds the stream's length; the forced prefix may hold up to 8 ids per second of audio plus `max_new_tokens`.
    pub fn open_stream(&self, max_samples: usize, lang_ids: Option<&[i64]>, rollback_ids: usize, unfixed_pushes: usize)
                       -> Result<B200Stream<'_>> {
        let m = self.max_new_tokens;
        let lang = lang_ids.map(|v| v.to_vec());
        let max_lang = lang.as_ref().map_or(0, |v| v.len()) + (max_samples * 8 + 15_999) / 16_000 + m;
        let mut session = ptr::null_mut();
        check(unsafe {
            ffi::asrb_session_create_ex(self.model.0, 1, max_samples.max(201) as i64, max_lang as i32, 0, m as i32, &mut session)
        })?;
        let session = Session(session);
        check(unsafe { ffi::asrb_stream_open(session.0, 1, rollback_ids as i32, unfixed_pushes as i32) })?;
        Ok(B200Stream { session, lang, max_ids: max_lang + m, max_new_tokens: m, _engine: self })
    }

    /// Long recordings: 16 kHz mono f32 `samples` of any length are cut on the GPU at the quietest 100 ms window of
    /// the last `search_samples` before every `max_segment_samples` (`asrb_segment_long`; both multiples of 160,
    /// `max_segment_samples` >= 80000, 32000 <= `search_samples` <= `max_segment_samples` / 2), and the segments are
    /// decoded as views of the ingested audio (`asrb_transcribe_segments`) in batches of up to `batch` segments.
    /// Returns the segments in time order as (start, end in samples, ids); `max_new_tokens` applies per segment.
    pub fn transcribe_long(&self, samples: &[f32], lang_ids: Option<&[i64]>, max_segment_samples: usize, search_samples: usize,
                           batch: usize) -> Result<Vec<(i64, i64, Vec<i64>)>> {
        if batch == 0 { return Err(anyhow!("batch must be >= 1")); }
        let session = self.session_for_slots(max_segment_samples.min(samples.len()).max(201), batch)?;
        let pcm = [samples.as_ptr() as *const std::os::raw::c_void];
        let (frames, chans, rate, fmt) = ([samples.len() as i64], [1i32], [16000i32], [1i32]);   // ASRB_PCM_F32
        let mut n = 0i64;
        check(unsafe { ffi::asrb_ingest_long(session, pcm.as_ptr(), frames.as_ptr(), chans.as_ptr(), rate.as_ptr(), fmt.as_ptr(), 1, &mut n) })?;
        let mut cap = 64usize;
        let (starts, ends) = loop {
            let mut nseg = 0i32;
            let (mut st, mut en) = (vec![0i64; cap], vec![0i64; cap]);
            let status = unsafe {
                ffi::asrb_segment_long(session, max_segment_samples as i64, search_samples as i64, cap as i32, &mut nseg,
                                       st.as_mut_ptr(), en.as_mut_ptr())
            };
            if status == ffi::ASRB_ERR_INVALID && nseg as usize > cap { cap = nseg as usize; continue; }
            check(status)?;
            st.truncate(nseg as usize);
            en.truncate(nseg as usize);
            break (st, en);
        };
        let m = self.max_new_tokens;
        let mut out = Vec::with_capacity(starts.len());
        for w0 in (0..starts.len()).step_by(batch) {
            let k = batch.min(starts.len() - w0);
            let files = vec![0i32; k];
            let lp = vec![lang_ids.map_or(ptr::null(), |v| v.as_ptr()); k];
            let ll = vec![lang_ids.map_or(0, |v| v.len() as i32); k];
            let mut ids = vec![0i32; k * m];
            let mut lens = vec![0i32; k];
            check(unsafe {
                ffi::asrb_transcribe_segments(session, k as i32, files.as_ptr(), starts[w0..].as_ptr(), ends[w0..].as_ptr(),
                                              lp.as_ptr(), ll.as_ptr(), m as i32, ids.as_mut_ptr(), lens.as_mut_ptr())
            })?;
            for j in 0..k {
                out.push((starts[w0 + j], ends[w0 + j], ids[j * m..j * m + lens[j] as usize].iter().map(|&t| t as i64).collect()));
            }
        }
        Ok(out)
    }
}

/// A live stream from `B200Engine::open_stream`; its session is freed on drop.
pub struct B200Stream<'a> {
    session: Session,
    lang: Option<Vec<i64>>,
    max_ids: usize,
    max_new_tokens: usize,
    _engine: &'a B200Engine,
}

impl B200Stream<'_> {
    /// Appends `samples` (the last push sets `is_final`) and returns (hypothesis ids, fixed length): the first `fixed`
    /// ids are forced into every later hypothesis of the stream.
    pub fn push(&mut self, samples: &[f32], is_final: bool) -> Result<(Vec<i64>, usize)> {
        let (ptrs, n, fin) = ([samples.as_ptr()], [samples.len() as i64], [is_final as i32]);
        let lp = [self.lang.as_ref().map_or(ptr::null(), |v| v.as_ptr())];
        let ll = [self.lang.as_ref().map_or(0, |v| v.len() as i32)];
        let mut hyp = vec![0i32; self.max_ids];
        let (mut len, mut fixed) = (0i32, 0i32);
        check(unsafe {
            ffi::asrb_stream_push(self.session.0, 1, ptrs.as_ptr(), n.as_ptr(), fin.as_ptr(), lp.as_ptr(), ll.as_ptr(),
                                  self.max_new_tokens as i32, self.max_ids as i32, hyp.as_mut_ptr(), &mut len, &mut fixed)
        })?;
        Ok((hyp[..len as usize].iter().map(|&t| t as i64).collect(), fixed as usize))
    }

    /// Back to an empty stream (after a final push, or to start over).
    pub fn reset(&mut self) -> Result<()> { check(unsafe { ffi::asrb_stream_reset(self.session.0, 0) }) }
}
