//! `bio_b200::alignment::{pairwise, distance}` -- the rust-bio 4.0.1 pairwise and distance APIs on an H100.
//!
//! NOT COMPILED BY THIS REPOSITORY'S BUILD (it needs no Rust toolchain).  It is the binding a
//! maintainer adds next to `bio`: same type and method names as
//! `bio::alignment::pairwise::{MIN_SCORE, MatchFunc, MatchParams, Scoring, Aligner}`
//! (rust-bio src/alignment/pairwise/mod.rs:174-1015) plus `*_batch` methods; every method goes
//! through the C ABI of `include/b200align.h` -- there is no CPU implementation behind it.
//!
//! ```ignore
//! // before:  use bio::alignment::pairwise::*;
//! use bio_b200::alignment::pairwise::*;
//! let score = |a: u8, b: u8| if a == b { 1i32 } else { -1i32 };
//! let mut aligner = Aligner::with_capacity(150, 150, -5, -1, &score);
//! let alns = aligner.local_batch(&pairs);          // Vec<bio_types::alignment::Alignment>
//! let one = aligner.local(x, y);                   // a batch of one
//! ```
#![allow(non_camel_case_types, non_snake_case)]

pub mod alignment {
    pub use bio_types::alignment::{Alignment, AlignmentMode, AlignmentOperation};

    pub mod pairwise {
        use super::{Alignment, AlignmentMode, AlignmentOperation};
        use std::ffi::CStr;
        use std::os::raw::{c_char, c_void};

        /// mod.rs:174
        pub const MIN_SCORE: i32 = -858_993_459;

        // ---------------------------------------------------------------- FFI (include/b200align.h)
        #[repr(C)]
        struct b2a_scoring {
            gap_open: i32,
            gap_extend: i32,
            xclip_prefix: i32,
            xclip_suffix: i32,
            yclip_prefix: i32,
            yclip_suffix: i32,
            match_score: i32,
            mismatch_score: i32,
            has_match_scores: i32,
            table: *const i32,
            alphabet: *const u8,
            alphabet_len: u32,
        }
        #[repr(C)]
        struct b2a_pairs {
            seq_blob: *const u8,
            x_off: *const u64,
            x_len: *const u32,
            y_off: *const u64,
            y_len: *const u32,
            blob_bytes: u64,
            n_pairs: u64,
        }
        #[repr(C)]
        struct b2a_results {
            score: *mut i32,
            xstart: *mut u32,
            xend: *mut u32,
            ystart: *mut u32,
            yend: *mut u32,
            ops_off: *mut u64,
            ops: *mut u8,
            ops_capacity: u64,
            clip_len: *mut u32,
            status: *mut u32, // per-pair B2A_PAIR_* codes; null = a failing pair fails the batch (-> panic, like the reference)
        }
        #[link(name = "b200align")]
        extern "C" {
            fn b2a_engine_create(out: *mut *mut c_void, device_id: i32) -> i32;
            // every visible GPU from this one process (include/b200align.h: b2a_multi_*)
            fn b2a_multi_create(out: *mut *mut c_void, device_ids: *const i32, n_devices: i32) -> i32;
            fn b2a_multi_destroy(m: *mut c_void) -> i32;
            fn b2a_multi_last_error(m: *const c_void) -> *const c_char;
            fn b2a_multi_align_batch(
                m: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                pairs: *const b2a_pairs,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
            fn b2a_multi_align_batch_banded(
                m: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                k: u32,
                w: u32,
                pairs: *const b2a_pairs,
                hints: *const b2a_band_hints,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
            fn b2a_multi_align_batch_scores(
                m: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                pairs: *const b2a_pairs,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
            fn b2a_multi_align_batch_banded_scores(
                m: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                k: u32,
                w: u32,
                pairs: *const b2a_pairs,
                hints: *const b2a_band_hints,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
            fn b2a_engine_destroy(e: *mut c_void) -> i32;
            fn b2a_last_error(e: *const c_void) -> *const c_char;
            fn b2a_engine_set_traceback_recompute(e: *mut c_void, on: i32) -> i32;
            #[allow(dead_code)]
            fn b2a_engine_last_recompute(e: *const c_void, pairs: *mut u64, windows: *mut u64, windows_filled: *mut u64) -> i32;
            fn b2a_align_batch(
                e: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                pairs: *const b2a_pairs,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
            fn b2a_align_batch_scores(
                e: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                pairs: *const b2a_pairs,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
            fn b2a_align_batch_banded(
                e: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                k: u32,
                w: u32,
                pairs: *const b2a_pairs,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
            fn b2a_align_batch_banded_hinted(
                e: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                k: u32,
                w: u32,
                pairs: *const b2a_pairs,
                hints: *const b2a_band_hints,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
            fn b2a_align_batch_banded_scores(
                e: *mut c_void,
                mode: i32,
                scoring: *const b2a_scoring,
                k: u32,
                w: u32,
                pairs: *const b2a_pairs,
                hints: *const b2a_band_hints,
                results: *mut b2a_results,
                stats: *mut c_void,
            ) -> i32;
        }
        #[repr(C)]
        struct b2a_band_hints {
            match_off: *const u64,
            match_xy: *const u32,
            path_off: *const u64,
            path_idx: *const u32,
            allowed_mismatches: i32,
            use_lcskpp_union: i32,
        }

        /// What a banded call adds to `Aligner::batch`: k, w and (banded.rs:294-401) the caller's band inputs.
        pub(crate) struct BandedCall<'a> {
            pub k: u32,
            pub w: u32,
            pub matches: Option<&'a [&'a [(u32, u32)]]>,
            pub paths: Option<&'a [&'a [usize]]>,
            pub allowed_mismatches: Option<usize>,
            pub use_lcskpp_union: bool,
        }

        // ---------------------------------------------------------------- scoring, mod.rs:177-429
        pub trait MatchFunc {
            fn score(&self, a: u8, b: u8) -> i32;
        }

        #[derive(Default, Copy, Clone, Eq, PartialEq, Ord, PartialOrd, Hash, Debug)]
        pub struct MatchParams {
            pub match_score: i32,
            pub mismatch_score: i32,
        }
        impl MatchParams {
            pub fn new(match_score: i32, mismatch_score: i32) -> Self {
                assert!(match_score >= 0, "match_score can't be negative");
                assert!(mismatch_score <= 0, "mismatch_score can't be positive");
                MatchParams { match_score, mismatch_score }
            }
        }
        impl MatchFunc for MatchParams {
            fn score(&self, a: u8, b: u8) -> i32 {
                if a == b { self.match_score } else { self.mismatch_score }
            }
        }
        impl<F> MatchFunc for F
        where
            F: Fn(u8, u8) -> i32,
        {
            fn score(&self, a: u8, b: u8) -> i32 {
                (self)(a, b)
            }
        }

        #[derive(Default, Copy, Clone, Eq, PartialEq, Ord, PartialOrd, Hash, Debug)]
        pub struct Scoring<F: MatchFunc> {
            pub gap_open: i32,
            pub gap_extend: i32,
            pub match_fn: F,
            pub match_scores: Option<(i32, i32)>,
            pub xclip_prefix: i32,
            pub xclip_suffix: i32,
            pub yclip_prefix: i32,
            pub yclip_suffix: i32,
        }
        impl Scoring<MatchParams> {
            pub fn from_scores(gap_open: i32, gap_extend: i32, match_score: i32, mismatch_score: i32) -> Self {
                assert!(gap_open <= 0, "gap_open can't be positive");
                assert!(gap_extend <= 0, "gap_extend can't be positive");
                Scoring {
                    gap_open,
                    gap_extend,
                    match_fn: MatchParams::new(match_score, mismatch_score),
                    match_scores: Some((match_score, mismatch_score)),
                    xclip_prefix: MIN_SCORE,
                    xclip_suffix: MIN_SCORE,
                    yclip_prefix: MIN_SCORE,
                    yclip_suffix: MIN_SCORE,
                }
            }
        }
        impl<F: MatchFunc> Scoring<F> {
            pub fn new(gap_open: i32, gap_extend: i32, match_fn: F) -> Self {
                assert!(gap_open <= 0, "gap_open can't be positive");
                assert!(gap_extend <= 0, "gap_extend can't be positive");
                Scoring {
                    gap_open,
                    gap_extend,
                    match_fn,
                    match_scores: None,
                    xclip_prefix: MIN_SCORE,
                    xclip_suffix: MIN_SCORE,
                    yclip_prefix: MIN_SCORE,
                    yclip_suffix: MIN_SCORE,
                }
            }
            pub fn xclip(mut self, penalty: i32) -> Self {
                assert!(penalty <= 0, "Clipping penalty can't be positive");
                self.xclip_prefix = penalty;
                self.xclip_suffix = penalty;
                self
            }
            pub fn xclip_prefix(mut self, penalty: i32) -> Self {
                assert!(penalty <= 0, "Clipping penalty can't be positive");
                self.xclip_prefix = penalty;
                self
            }
            pub fn xclip_suffix(mut self, penalty: i32) -> Self {
                assert!(penalty <= 0, "Clipping penalty can't be positive");
                self.xclip_suffix = penalty;
                self
            }
            pub fn yclip(mut self, penalty: i32) -> Self {
                assert!(penalty <= 0, "Clipping penalty can't be positive");
                self.yclip_prefix = penalty;
                self.yclip_suffix = penalty;
                self
            }
            pub fn yclip_prefix(mut self, penalty: i32) -> Self {
                assert!(penalty <= 0, "Clipping penalty can't be positive");
                self.yclip_prefix = penalty;
                self
            }
            pub fn yclip_suffix(mut self, penalty: i32) -> Self {
                assert!(penalty <= 0, "Clipping penalty can't be positive");
                self.yclip_suffix = penalty;
                self
            }
        }

        // ---------------------------------------------------------------- Aligner, mod.rs:472-1015
        /// Holds the scoring and an engine handle (one CUDA device) instead of host scratch vectors.
        /// Not `Clone`/`Serialize` (documented API deviation, SURVEY section 5).
        pub struct Aligner<F: MatchFunc> {
            scoring: Scoring<F>,
            engine: *mut c_void,
            /// non-null after `on_all_gpus()`: `*_batch` calls are split over every visible GPU (one ncclAllGather
            /// reassembles them); the banded entry points stay on `engine`'s device
            multi: *mut c_void,
        }
        unsafe impl<F: MatchFunc + Send> Send for Aligner<F> {}

        /// What a `*_scores_batch` call returns per pair: `Alignment::{score, xend, yend}` (no start coordinates, no
        /// operations: those come out of the traceback, which a score-only batch does not keep).
        #[derive(Clone, Copy, Debug, PartialEq, Eq)]
        pub struct AlignmentScore {
            pub score: i32,
            pub xend: usize,
            pub yend: usize,
        }

        /// A batch in the C ABI's input layout (owned; `c_pairs` borrows it)
        struct PackedBatch {
            blob: Vec<u8>,
            x_off: Vec<u64>,
            y_off: Vec<u64>,
            x_len: Vec<u32>,
            y_len: Vec<u32>,
            table: Vec<i32>,
            alphabet: Vec<u8>,
        }

        impl PackedBatch {
            fn c_pairs(&self) -> b2a_pairs {
                b2a_pairs {
                    seq_blob: self.blob.as_ptr(),
                    x_off: self.x_off.as_ptr(),
                    x_len: self.x_len.as_ptr(),
                    y_off: self.y_off.as_ptr(),
                    y_len: self.y_len.as_ptr(),
                    blob_bytes: self.blob.len() as u64,
                    n_pairs: self.x_len.len() as u64,
                }
            }
        }

        impl<F: MatchFunc> Drop for Aligner<F> {
            fn drop(&mut self) {
                unsafe {
                    if !self.multi.is_null() {
                        b2a_multi_destroy(self.multi);
                    }
                    b2a_engine_destroy(self.engine)
                };
            }
        }

        const DEFAULT_ALIGNER_CAPACITY: usize = 200;

        impl<F: MatchFunc> Aligner<F> {
            pub fn new(gap_open: i32, gap_extend: i32, match_fn: F) -> Self {
                Aligner::with_capacity(DEFAULT_ALIGNER_CAPACITY, DEFAULT_ALIGNER_CAPACITY, gap_open, gap_extend, match_fn)
            }
            pub fn with_capacity(_m: usize, _n: usize, gap_open: i32, gap_extend: i32, match_fn: F) -> Self {
                assert!(gap_open <= 0, "gap_open can't be positive");
                assert!(gap_extend <= 0, "gap_extend can't be positive");
                Self::make(Scoring::new(gap_open, gap_extend, match_fn))
            }
            pub fn with_scoring(scoring: Scoring<F>) -> Self {
                Aligner::with_capacity_and_scoring(DEFAULT_ALIGNER_CAPACITY, DEFAULT_ALIGNER_CAPACITY, scoring)
            }
            pub fn with_capacity_and_scoring(_m: usize, _n: usize, scoring: Scoring<F>) -> Self {
                assert!(scoring.gap_open <= 0, "gap_open can't be positive");
                assert!(scoring.gap_extend <= 0, "gap_extend can't be positive");
                assert!(scoring.xclip_prefix <= 0, "Clipping penalty (x prefix) can't be positive");
                assert!(scoring.xclip_suffix <= 0, "Clipping penalty (x suffix) can't be positive");
                assert!(scoring.yclip_prefix <= 0, "Clipping penalty (y prefix) can't be positive");
                assert!(scoring.yclip_suffix <= 0, "Clipping penalty (y suffix) can't be positive");
                Self::make(scoring)
            }
            fn make(scoring: Scoring<F>) -> Self {
                let mut engine: *mut c_void = std::ptr::null_mut();
                let device = std::env::var("B2A_DEVICE").ok().and_then(|v| v.parse().ok()).unwrap_or(0);
                let rc = unsafe { b2a_engine_create(&mut engine, device) };
                assert!(rc == 0, "b200align: no usable sm_90 (H100) device (rc = {}); there is no CPU fallback", rc);
                Aligner { scoring, engine, multi: std::ptr::null_mut() }
            }

            /// Use every visible GPU for the `*_batch` methods (not part of rust-bio's API: its Aligner is a
            /// single-threaded CPU object).  Panics if the devices cannot be opened.
            pub fn on_all_gpus(mut self) -> Self {
                let mut m: *mut c_void = std::ptr::null_mut();
                let rc = unsafe { b2a_multi_create(&mut m, std::ptr::null(), 0) };
                assert!(rc == 0, "b200align: cannot open every visible device (rc = {})", rc);
                self.multi = m;
                self
            }

            /// Align a pair whose traceback is above the engine's traceback budget (default 60 % of free HBM) by
            /// recomputing it one window of strips at a time, instead of refusing it (not part of rust-bio's API).
            /// Results are the same; such a pair costs at least one more fill.  Applies to this Aligner's engine;
            /// `on_all_gpus()` batches keep each device's default.
            pub fn with_traceback_recompute(self) -> Self {
                let rc = unsafe { b2a_engine_set_traceback_recompute(self.engine, 1) };
                assert!(rc == 0, "b200align: cannot set traceback recompute (rc = {})", rc);
                self
            }

            /// Text of the last failure: of the multi-GPU handle after `on_all_gpus()`, else of the engine.
            fn error_text(&self) -> String {
                let p = if self.multi.is_null() {
                    unsafe { b2a_last_error(self.engine) }
                } else {
                    unsafe { b2a_multi_last_error(self.multi) }
                };
                unsafe { CStr::from_ptr(p) }.to_string_lossy().into_owned()
            }

            /// The batch in the C ABI's input layout: 16-byte aligned slots (x then y per pair), and the MatchFunc
            /// tabulated over the symbols present (mod.rs:221-228 allows any closure).
            fn pack(&self, pairs: &[(&[u8], &[u8])]) -> PackedBatch {
                let n = pairs.len();
                let mut x_off = Vec::with_capacity(n);
                let mut y_off = Vec::with_capacity(n);
                let mut x_len = Vec::with_capacity(n);
                let mut y_len = Vec::with_capacity(n);
                let mut blob: Vec<u8> = Vec::new();
                let mut present = [false; 256];
                for (x, y) in pairs {
                    for s in [x, y] {
                        while blob.len() % 16 != 0 {
                            blob.push(0);
                        }
                        if std::ptr::eq(*s, *x) { x_off.push(blob.len() as u64) } else { y_off.push(blob.len() as u64) }
                        blob.extend_from_slice(s);
                        for &b in s.iter() {
                            present[b as usize] = true;
                        }
                    }
                    x_len.push(x.len() as u32);
                    y_len.push(y.len() as u32);
                }
                let alphabet: Vec<u8> = (0..=255u8).filter(|b| present[*b as usize]).collect();
                let mut table = vec![0i32; 256 * 256];
                for &a in &alphabet {
                    for &b in &alphabet {
                        table[a as usize * 256 + b as usize] = self.scoring.match_fn.score(a, b);
                    }
                }
                PackedBatch { blob, x_off, y_off, x_len, y_len, table, alphabet }
            }

            fn c_scoring(&self, pb: &PackedBatch) -> b2a_scoring {
                let (ms, mm) = self.scoring.match_scores.unwrap_or((0, 0));
                b2a_scoring {
                    gap_open: self.scoring.gap_open,
                    gap_extend: self.scoring.gap_extend,
                    xclip_prefix: self.scoring.xclip_prefix,
                    xclip_suffix: self.scoring.xclip_suffix,
                    yclip_prefix: self.scoring.yclip_prefix,
                    yclip_suffix: self.scoring.yclip_suffix,
                    match_score: ms,
                    mismatch_score: mm,
                    has_match_scores: self.scoring.match_scores.is_some() as i32,
                    table: pb.table.as_ptr(),
                    alphabet: pb.alphabet.as_ptr(),
                    alphabet_len: pb.alphabet.len() as u32,
                }
            }

            /// Aligner::custom / global / semiglobal / local over a batch (mode = B2A_MODE_*).
            pub(crate) fn batch(&mut self, mode: i32, banded: Option<BandedCall>, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> {
                let n = pairs.len();
                let pb = self.pack(pairs);
                let (cs, cp) = (self.c_scoring(&pb), pb.c_pairs());
                let cap: u64 = pairs.iter().map(|(x, y)| (x.len() + y.len() + 4) as u64).sum();
                let mut score = vec![0i32; n];
                let (mut xs, mut xe, mut ys, mut ye) = (vec![0u32; n], vec![0u32; n], vec![0u32; n], vec![0u32; n]);
                let mut ops_off = vec![0u64; n + 1];
                let mut ops = vec![0u8; cap as usize + 1];
                let mut clip = vec![0u32; 4 * n.max(1)];
                let mut res = b2a_results {
                    score: score.as_mut_ptr(),
                    xstart: xs.as_mut_ptr(),
                    xend: xe.as_mut_ptr(),
                    ystart: ys.as_mut_ptr(),
                    yend: ye.as_mut_ptr(),
                    ops_off: ops_off.as_mut_ptr(),
                    ops: ops.as_mut_ptr(),
                    ops_capacity: cap + 1,
                    clip_len: clip.as_mut_ptr(),
                    status: std::ptr::null_mut(),
                };
                let is_banded = banded.is_some();
                let rc = match banded {
                    None if !self.multi.is_null() => {
                        let rc = unsafe { b2a_multi_align_batch(self.multi, mode, &cs, &cp, &mut res, std::ptr::null_mut()) };
                        if rc != 0 {
                            let msg = unsafe { CStr::from_ptr(b2a_multi_last_error(self.multi)) }.to_string_lossy().into_owned();
                            panic!("{}", msg);
                        }
                        rc
                    }
                    None => unsafe { b2a_align_batch(self.engine, mode, &cs, &cp, &mut res, std::ptr::null_mut()) },
                    Some(BandedCall { k, w, matches: None, .. }) if !self.multi.is_null() => unsafe {
                        b2a_multi_align_batch_banded(self.multi, mode, &cs, k, w, &cp, std::ptr::null(), &mut res,
                                                     std::ptr::null_mut())
                    },
                    Some(BandedCall { k, w, matches: None, .. }) => unsafe {
                        b2a_align_batch_banded(self.engine, mode, &cs, k, w, &cp, &mut res, std::ptr::null_mut())
                    },
                    Some(BandedCall { k, w, matches: Some(ms), paths, allowed_mismatches, use_lcskpp_union }) => {
                        // CSR form of the per-pair matches (and paths), include/b200align.h b2a_band_hints
                        assert!(ms.len() == n, "one match list per pair");
                        let mut match_off = vec![0u64; n + 1];
                        let mut match_xy: Vec<u32> = Vec::new();
                        for (p, m) in ms.iter().enumerate() {
                            for &(a, b) in m.iter() {
                                match_xy.push(a);
                                match_xy.push(b);
                            }
                            match_off[p + 1] = (match_xy.len() / 2) as u64;
                        }
                        match_xy.push(0); // never a dangling pointer for an empty list
                        let mut path_off = vec![0u64; n + 1];
                        let mut path_idx: Vec<u32> = Vec::new();
                        if let Some(ps) = paths {
                            assert!(ps.len() == n, "one path per pair");
                            for (p, path) in ps.iter().enumerate() {
                                path_idx.extend(path.iter().map(|&i| i as u32));
                                path_off[p + 1] = path_idx.len() as u64;
                            }
                        }
                        path_idx.push(0);
                        let h = b2a_band_hints {
                            match_off: match_off.as_ptr(),
                            match_xy: match_xy.as_ptr(),
                            path_off: if paths.is_some() { path_off.as_ptr() } else { std::ptr::null() },
                            path_idx: if paths.is_some() { path_idx.as_ptr() } else { std::ptr::null() },
                            allowed_mismatches: allowed_mismatches.map(|v| v as i32).unwrap_or(-1),
                            use_lcskpp_union: use_lcskpp_union as i32,
                        };
                        if !self.multi.is_null() {
                            unsafe { b2a_multi_align_batch_banded(self.multi, mode, &cs, k, w, &cp, &h, &mut res, std::ptr::null_mut()) }
                        } else {
                            unsafe {
                                b2a_align_batch_banded_hinted(self.engine, mode, &cs, k, w, &cp, &h, &mut res, std::ptr::null_mut())
                            }
                        }
                    }
                };
                if rc != 0 {
                    let msg = self.error_text();
                    panic!("{}", msg); // the reference panics on the same conditions (assert!, mod.rs:905)
                }
                let amode = match mode {
                    1 => AlignmentMode::Global,
                    2 => AlignmentMode::Semiglobal,
                    3 => AlignmentMode::Local,
                    _ => AlignmentMode::Custom,
                };
                (0..n)
                    .map(|p| {
                        let mut k = 0;
                        let operations = ops[ops_off[p] as usize..ops_off[p + 1] as usize]
                            .iter()
                            .map(|c| match c {
                                0 => AlignmentOperation::Match,
                                1 => AlignmentOperation::Subst,
                                2 => AlignmentOperation::Del,
                                3 => AlignmentOperation::Ins,
                                4 => {
                                    k += 1;
                                    AlignmentOperation::Xclip(clip[4 * p + k - 1] as usize)
                                }
                                _ => {
                                    k += 1;
                                    AlignmentOperation::Yclip(clip[4 * p + k - 1] as usize)
                                }
                            })
                            .collect();
                        // banded.rs:407-420: a band above MAX_CELLS returns the empty alignment (score MIN_SCORE,
                        // xlen = ylen = 0); global/semiglobal/local then overwrite only `.mode` (banded.rs:889-890)
                        let operations: Vec<AlignmentOperation> = operations;
                        let refused = is_banded && score[p] == MIN_SCORE && operations.is_empty();
                        Alignment {
                            score: score[p],
                            ystart: ys[p] as usize,
                            xstart: xs[p] as usize,
                            yend: ye[p] as usize,
                            xend: xe[p] as usize,
                            ylen: if refused { 0 } else { pairs[p].1.len() },
                            xlen: if refused { 0 } else { pairs[p].0.len() },
                            operations,
                            mode: amode,
                        }
                    })
                    .collect()
            }

            pub fn custom_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> { self.batch(0, None, pairs) }
            pub fn global_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> { self.batch(1, None, pairs) }
            pub fn semiglobal_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> { self.batch(2, None, pairs) }
            pub fn local_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> { self.batch(3, None, pairs) }

            /// Alignment::{score, xend, yend} of each pair without the traceback (b2a_align_batch_scores, or with
            /// banded = Some((k, w)) b2a_align_batch_banded_scores), on this aligner's device, or split over every
            /// device after `on_all_gpus()` (the b2a_multi_* forms).  Panics where the full call would (a pair the
            /// reference panics on).
            pub(crate) fn scores_batch(&mut self, mode: i32, banded: Option<(u32, u32)>, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> {
                let n = pairs.len();
                let pb = self.pack(pairs);
                let (cs, cp) = (self.c_scoring(&pb), pb.c_pairs());
                let mut score = vec![0i32; n.max(1)];
                let (mut xe, mut ye) = (vec![0u32; n.max(1)], vec![0u32; n.max(1)]);
                let mut res = b2a_results {
                    score: score.as_mut_ptr(),
                    xstart: std::ptr::null_mut(),
                    xend: xe.as_mut_ptr(),
                    ystart: std::ptr::null_mut(),
                    yend: ye.as_mut_ptr(),
                    ops_off: std::ptr::null_mut(),
                    ops: std::ptr::null_mut(),
                    ops_capacity: 0,
                    clip_len: std::ptr::null_mut(),
                    status: std::ptr::null_mut(),
                };
                let multi = !self.multi.is_null();
                let rc = match banded {
                    None if multi => unsafe {
                        b2a_multi_align_batch_scores(self.multi, mode, &cs, &cp, &mut res, std::ptr::null_mut())
                    },
                    None => unsafe { b2a_align_batch_scores(self.engine, mode, &cs, &cp, &mut res, std::ptr::null_mut()) },
                    Some((k, w)) if multi => unsafe {
                        b2a_multi_align_batch_banded_scores(self.multi, mode, &cs, k, w, &cp, std::ptr::null(), &mut res,
                                                            std::ptr::null_mut())
                    },
                    Some((k, w)) => unsafe {
                        b2a_align_batch_banded_scores(self.engine, mode, &cs, k, w, &cp, std::ptr::null(), &mut res,
                                                      std::ptr::null_mut())
                    },
                };
                if rc != 0 {
                    panic!("{}", self.error_text());
                }
                (0..n).map(|p| AlignmentScore { score: score[p], xend: xe[p] as usize, yend: ye[p] as usize }).collect()
            }

            pub fn custom_scores_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> { self.scores_batch(0, None, pairs) }
            pub fn global_scores_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> { self.scores_batch(1, None, pairs) }
            pub fn semiglobal_scores_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> { self.scores_batch(2, None, pairs) }
            pub fn local_scores_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> { self.scores_batch(3, None, pairs) }

            /// mod.rs:591
            pub fn custom(&mut self, x: &[u8], y: &[u8]) -> Alignment { self.batch(0, None, &[(x, y)]).remove(0) }
            /// mod.rs:925
            pub fn global(&mut self, x: &[u8], y: &[u8]) -> Alignment { self.batch(1, None, &[(x, y)]).remove(0) }
            /// mod.rs:954
            pub fn semiglobal(&mut self, x: &[u8], y: &[u8]) -> Alignment { self.batch(2, None, &[(x, y)]).remove(0) }
            /// mod.rs:986
            pub fn local(&mut self, x: &[u8], y: &[u8]) -> Alignment { self.batch(3, None, &[(x, y)]).remove(0) }
        }

        // ------------------------------------------------------------ TracebackCell, mod.rs:1026-1114
        /// The reference's public packed traceback cell: three 4-bit move codes, I in the low nibble, then D, then S.
        /// The engine keeps its own 4-bit traceback on the device; this host type exists for callers that named it.
        #[derive(Default, Copy, Clone, Eq, PartialEq, Ord, PartialOrd, Hash, Debug)]
        pub struct TracebackCell {
            v: u16,
        }
        #[derive(Copy, Clone)]
        enum Layer {
            I = 0,
            D = 4,
            S = 8,
        }
        const LARGEST_MOVE: u16 = 8; // TB_YCLIP_SUFFIX
        impl TracebackCell {
            pub fn new() -> TracebackCell {
                TracebackCell { v: 0 }
            }
            fn put(&mut self, layer: Layer, code: u16) {
                assert!(code <= LARGEST_MOVE, "Expected a value <= TB_MAX while setting traceback bits");
                let shift = layer as u16;
                self.v &= !(0xF << shift);
                self.v |= code << shift;
            }
            fn take(self, layer: Layer) -> u16 {
                (self.v >> (layer as u16)) & 0xF
            }
            pub fn set_i_bits(&mut self, value: u16) { self.put(Layer::I, value) }
            pub fn set_d_bits(&mut self, value: u16) { self.put(Layer::D, value) }
            pub fn set_s_bits(&mut self, value: u16) { self.put(Layer::S, value) }
            pub fn get_i_bits(self) -> u16 { self.take(Layer::I) }
            pub fn get_d_bits(self) -> u16 { self.take(Layer::D) }
            pub fn get_s_bits(self) -> u16 { self.take(Layer::S) }
            pub fn set_all(&mut self, value: u16) {
                for layer in [Layer::I, Layer::D, Layer::S] {
                    self.put(layer, value);
                }
            }
        }

        // ------------------------------------------------------------ banded::Aligner, banded.rs:122-1004
        pub mod banded {
            use super::{Alignment, AlignmentScore, BandedCall, MatchFunc, Scoring};

            /// Same constructors and methods as `bio::alignment::pairwise::banded::Aligner` (k = k-mer length,
            /// w = band half-width, banded.rs:150-267); every method is a batch of one, `*_batch` is the GPU form.
            pub struct Aligner<F: MatchFunc> {
                inner: super::Aligner<F>,
                k: usize,
                w: usize,
            }

            impl<F: MatchFunc> Aligner<F> {
                pub fn new(gap_open: i32, gap_extend: i32, match_fn: F, k: usize, w: usize) -> Self {
                    Aligner { inner: super::Aligner::new(gap_open, gap_extend, match_fn), k, w }
                }
                pub fn with_capacity(m: usize, n: usize, gap_open: i32, gap_extend: i32, match_fn: F, k: usize, w: usize) -> Self {
                    Aligner { inner: super::Aligner::with_capacity(m, n, gap_open, gap_extend, match_fn), k, w }
                }
                pub fn with_scoring(scoring: Scoring<F>, k: usize, w: usize) -> Self {
                    Aligner { inner: super::Aligner::with_scoring(scoring), k, w }
                }
                pub fn with_capacity_and_scoring(m: usize, n: usize, scoring: Scoring<F>, k: usize, w: usize) -> Self {
                    Aligner { inner: super::Aligner::with_capacity_and_scoring(m, n, scoring), k, w }
                }
                /// Split the `*_batch` and `*_scores_batch` calls over every visible GPU (super::Aligner::on_all_gpus;
                /// not part of rust-bio's API).  Panics if the devices cannot be opened.
                pub fn on_all_gpus(mut self) -> Self {
                    self.inner = self.inner.on_all_gpus();
                    self
                }
                pub fn get_mut_scoring(&mut self) -> &mut Scoring<F> {
                    &mut self.inner.scoring
                }
                fn call<'a>(&self) -> BandedCall<'a> {
                    BandedCall { k: self.k as u32, w: self.w as u32, matches: None, paths: None, allowed_mismatches: None, use_lcskpp_union: false }
                }

                pub fn custom_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> { let c = self.call(); self.inner.batch(0, Some(c), pairs) }
                pub fn global_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> { let c = self.call(); self.inner.batch(1, Some(c), pairs) }
                pub fn semiglobal_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> { let c = self.call(); self.inner.batch(2, Some(c), pairs) }
                pub fn local_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<Alignment> { let c = self.call(); self.inner.batch(3, Some(c), pairs) }
                /// Alignment::{score, xend, yend} of each pair without the traceback (b2a_align_batch_banded_scores):
                /// what the `*_batch` form returns in those fields; a band above MAX_CELLS gives (MIN_SCORE, 0, 0).
                pub fn custom_scores_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> { let (k, w) = (self.k as u32, self.w as u32); self.inner.scores_batch(0, Some((k, w)), pairs) }
                pub fn global_scores_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> { let (k, w) = (self.k as u32, self.w as u32); self.inner.scores_batch(1, Some((k, w)), pairs) }
                pub fn semiglobal_scores_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> { let (k, w) = (self.k as u32, self.w as u32); self.inner.scores_batch(2, Some((k, w)), pairs) }
                pub fn local_scores_batch(&mut self, pairs: &[(&[u8], &[u8])]) -> Vec<AlignmentScore> { let (k, w) = (self.k as u32, self.w as u32); self.inner.scores_batch(3, Some((k, w)), pairs) }
                /// banded.rs:282
                pub fn custom(&mut self, x: &[u8], y: &[u8]) -> Alignment { self.custom_batch(&[(x, y)]).remove(0) }
                /// banded.rs:872
                pub fn global(&mut self, x: &[u8], y: &[u8]) -> Alignment { self.global_batch(&[(x, y)]).remove(0) }
                /// banded.rs:901
                pub fn semiglobal(&mut self, x: &[u8], y: &[u8]) -> Alignment { self.semiglobal_batch(&[(x, y)]).remove(0) }
                /// banded.rs:975
                pub fn local(&mut self, x: &[u8], y: &[u8]) -> Alignment { self.local_batch(&[(x, y)]).remove(0) }

                /// banded.rs:294 / 938: the prehash of y only spares the reference its own hashing; the matches
                /// (find_kmer_matches_seq2_hashed) and therefore the results are those of custom / semiglobal.
                pub fn custom_with_prehash<H>(&mut self, x: &[u8], y: &[u8], _y_kmer_hash: &H) -> Alignment { self.custom(x, y) }
                pub fn semiglobal_with_prehash<H>(&mut self, x: &[u8], y: &[u8], _y_kmer_hash: &H) -> Alignment { self.semiglobal(x, y) }

                /// banded.rs:313
                pub fn custom_with_matches(&mut self, x: &[u8], y: &[u8], matches: &[(u32, u32)]) -> Alignment {
                    self.custom_with_matches_batch(&[(x, y)], &[matches]).remove(0)
                }
                pub fn custom_with_matches_batch(&mut self, pairs: &[(&[u8], &[u8])], matches: &[&[(u32, u32)]]) -> Vec<Alignment> {
                    let mut c = self.call();
                    c.matches = Some(matches);
                    self.inner.batch(0, Some(c), pairs)
                }
                /// banded.rs:338
                pub fn custom_with_expanded_matches(&mut self, x: &[u8], y: &[u8], matches: Vec<(u32, u32)>,
                                                    allowed_mismatches: Option<usize>, use_lcskpp_union: bool) -> Alignment {
                    self.custom_with_expanded_matches_batch(&[(x, y)], &[&matches[..]], allowed_mismatches, use_lcskpp_union).remove(0)
                }
                pub fn custom_with_expanded_matches_batch(&mut self, pairs: &[(&[u8], &[u8])], matches: &[&[(u32, u32)]],
                                                          allowed_mismatches: Option<usize>, use_lcskpp_union: bool) -> Vec<Alignment> {
                    let mut c = self.call();
                    c.matches = Some(matches);
                    c.allowed_mismatches = allowed_mismatches;
                    c.use_lcskpp_union = use_lcskpp_union;
                    self.inner.batch(0, Some(c), pairs)
                }
                /// banded.rs:391
                pub fn custom_with_match_path(&mut self, x: &[u8], y: &[u8], matches: &[(u32, u32)], path: &[usize]) -> Alignment {
                    self.custom_with_match_path_batch(&[(x, y)], &[matches], &[path]).remove(0)
                }
                pub fn custom_with_match_path_batch(&mut self, pairs: &[(&[u8], &[u8])], matches: &[&[(u32, u32)]],
                                                    paths: &[&[usize]]) -> Vec<Alignment> {
                    let mut c = self.call();
                    c.matches = Some(matches);
                    c.paths = Some(paths);
                    self.inner.batch(0, Some(c), pairs)
                }
            }
        }
    }

    // ---------------------------------------------------------------- distance, reference src/alignment/distance.rs
    /// `bio::alignment::distance` on the GPU: the reference's free functions (each a batch of one) and `*_batch`
    /// forms over a pair list, all on this thread's engine on device 0 (created on first use).
    pub mod distance {
        use std::cell::RefCell;
        use std::ffi::CStr;
        use std::os::raw::{c_char, c_void};

        /// B2A_DIST_NONE (include/b200align.h): no bound (k), or None (a bounded result)
        const DIST_NONE: u32 = 0xFFFF_FFFF;
        const PAIR_OK: u32 = 0;

        #[repr(C)]
        struct b2a_pairs {
            seq_blob: *const u8,
            x_off: *const u64,
            x_len: *const u32,
            y_off: *const u64,
            y_len: *const u32,
            blob_bytes: u64,
            n_pairs: u64,
        }
        #[link(name = "b200align")]
        extern "C" {
            fn b2a_engine_create(out: *mut *mut c_void, device_id: i32) -> i32;
            fn b2a_engine_destroy(e: *mut c_void) -> i32;
            fn b2a_last_error(e: *const c_void) -> *const c_char;
            fn b2a_levenshtein_batch(e: *mut c_void, k: u32, pairs: *const b2a_pairs, distance: *mut u32,
                                     stats: *mut c_void) -> i32;
            fn b2a_hamming_batch(e: *mut c_void, pairs: *const b2a_pairs, distance: *mut u32, status: *mut u32,
                                 stats: *mut c_void) -> i32;
        }

        struct Engine(*mut c_void);
        impl Drop for Engine {
            fn drop(&mut self) {
                if !self.0.is_null() {
                    unsafe { b2a_engine_destroy(self.0) };
                }
            }
        }
        thread_local! {
            static ENGINE: RefCell<Engine> = RefCell::new(Engine(std::ptr::null_mut()));
        }

        /// The pairs back to back in one blob (the kernels take any offsets)
        struct Batch {
            blob: Vec<u8>,
            x_off: Vec<u64>,
            y_off: Vec<u64>,
            x_len: Vec<u32>,
            y_len: Vec<u32>,
        }
        impl Batch {
            fn new(pairs: &[(&[u8], &[u8])]) -> Self {
                let mut b = Batch { blob: Vec::new(), x_off: Vec::new(), y_off: Vec::new(), x_len: Vec::new(), y_len: Vec::new() };
                for (x, y) in pairs {
                    assert!(x.len() < (1usize << 31) && y.len() < (1usize << 31), "b200align: a sequence longer than 2^31 - 1");
                    b.x_off.push(b.blob.len() as u64);
                    b.blob.extend_from_slice(x);
                    b.y_off.push(b.blob.len() as u64);
                    b.blob.extend_from_slice(y);
                    b.x_len.push(x.len() as u32);
                    b.y_len.push(y.len() as u32);
                }
                b
            }
            fn c_pairs(&self) -> b2a_pairs {
                b2a_pairs {
                    seq_blob: self.blob.as_ptr(),
                    x_off: self.x_off.as_ptr(),
                    x_len: self.x_len.as_ptr(),
                    y_off: self.y_off.as_ptr(),
                    y_len: self.y_len.as_ptr(),
                    blob_bytes: self.blob.len() as u64,
                    n_pairs: self.x_len.len() as u64,
                }
            }
        }

        /// Run `f` on this thread's engine; a failing call panics with the engine's error text (no CPU fallback).
        /// `pattern_matching::myers` and `stats::pairhmm` share the engine.
        pub(crate) fn with_engine(f: impl FnOnce(*mut c_void) -> i32) {
            ENGINE.with(|cell| {
                let mut eng = cell.borrow_mut();
                if eng.0.is_null() {
                    let mut h: *mut c_void = std::ptr::null_mut();
                    let rc = unsafe { b2a_engine_create(&mut h, 0) };
                    assert!(rc == 0, "b200align: cannot create an engine on device 0 (rc = {})", rc);
                    eng.0 = h;
                }
                let rc = f(eng.0);
                if rc != 0 {
                    let msg = unsafe { CStr::from_ptr(b2a_last_error(eng.0)) }.to_string_lossy().into_owned();
                    panic!("b200align: {} (rc = {})", msg, rc);
                }
            })
        }

        fn levenshtein_k(pairs: &[(&[u8], &[u8])], k: u32) -> Vec<u32> {
            let mut out = vec![0u32; pairs.len()];
            if pairs.is_empty() {
                return out;
            }
            let b = Batch::new(pairs);
            let cp = b.c_pairs();
            with_engine(|e| unsafe { b2a_levenshtein_batch(e, k, &cp, out.as_mut_ptr(), std::ptr::null_mut()) });
            out
        }

        /// Hamming distances of pairs already checked to have equal lengths
        fn hamming_equal(pairs: &[(&[u8], &[u8])]) -> Vec<u64> {
            let mut out = vec![0u32; pairs.len()];
            let mut status = vec![PAIR_OK; pairs.len()];
            if !pairs.is_empty() {
                let b = Batch::new(pairs);
                let cp = b.c_pairs();
                with_engine(|e| unsafe { b2a_hamming_batch(e, &cp, out.as_mut_ptr(), status.as_mut_ptr(), std::ptr::null_mut()) });
            }
            out.into_iter().map(u64::from).collect()
        }

        /// distance.rs:25-40; panics with the reference's message on unequal lengths (a batch: on the first such pair)
        pub fn hamming_batch(pairs: &[(&[u8], &[u8])]) -> Vec<u64> {
            for (x, y) in pairs {
                assert_eq!(x.len(), y.len(), "hamming distance cannot be calculated for texts of different length ({}!={})",
                           x.len(), y.len());
            }
            hamming_equal(pairs)
        }

        /// levenshtein over a batch (distance.rs:59-61)
        pub fn levenshtein_batch(pairs: &[(&[u8], &[u8])]) -> Vec<u32> {
            levenshtein_k(pairs, DIST_NONE)
        }

        pub fn hamming(alpha: &[u8], beta: &[u8]) -> u64 {
            hamming_batch(&[(alpha, beta)])[0]
        }

        pub fn levenshtein(alpha: &[u8], beta: &[u8]) -> u32 {
            levenshtein_batch(&[(alpha, beta)])[0]
        }

        /// distance.rs:63-173: the same values as the scalar functions
        pub mod simd {
            /// distance.rs:101-111, with simd::hamming's own panic message
            pub fn hamming_batch(pairs: &[(&[u8], &[u8])]) -> Vec<u64> {
                for (x, y) in pairs {
                    assert_eq!(x.len(), y.len(),
                               "simd hamming distance cannot be calculated for texts of different length ({}!={})",
                               x.len(), y.len());
                }
                super::hamming_equal(pairs)
            }

            pub fn levenshtein_batch(pairs: &[(&[u8], &[u8])]) -> Vec<u32> {
                super::levenshtein_batch(pairs)
            }

            /// distance.rs:165-172: per pair the distance if it is <= min(k, max(|x|, |y|)), else None
            pub fn bounded_levenshtein_batch(pairs: &[(&[u8], &[u8])], k: u32) -> Vec<Option<u32>> {
                let d = super::levenshtein_k(pairs, k);
                if k == super::DIST_NONE {
                    return d.into_iter().map(Some).collect();  // u32::MAX bounds nothing: every distance is Some
                }
                d.into_iter().map(|v| if v == super::DIST_NONE { None } else { Some(v) }).collect()
            }

            pub fn hamming(alpha: &[u8], beta: &[u8]) -> u64 {
                hamming_batch(&[(alpha, beta)])[0]
            }

            pub fn levenshtein(alpha: &[u8], beta: &[u8]) -> u32 {
                levenshtein_batch(&[(alpha, beta)])[0]
            }

            pub fn bounded_levenshtein(alpha: &[u8], beta: &[u8], k: u32) -> Option<u32> {
                bounded_levenshtein_batch(&[(alpha, beta)], k)[0]
            }
        }
    }
}

// ---------------------------------------------------------------- pattern matching, reference src/pattern_matching
/// `bio::pattern_matching` on the GPU: the Myers bit-parallel search (`myers`).
pub mod pattern_matching {
    /// `bio::pattern_matching::myers` (reference src/pattern_matching/myers): `Myers<u64>`, `Myers<u128>`,
    /// `long::Myers` and `MyersBuilder`, with the reference's `distance`, `find_all_end` and `find_best_end` (each a
    /// batch of one) and `*_batch` forms over many texts that store the pattern once, on the thread's engine of
    /// `alignment::distance`.  `find_all_end` returns the hits as a `Vec` rather than a lazy iterator.
    pub mod myers {
        use std::collections::HashMap;
        use std::marker::PhantomData;
        use std::os::raw::c_void;

        use crate::alignment::distance::with_engine;

        #[repr(C)]
        struct b2a_pairs {
            seq_blob: *const u8,
            x_off: *const u64,
            x_len: *const u32,
            y_off: *const u64,
            y_len: *const u32,
            blob_bytes: u64,
            n_pairs: u64,
        }
        #[repr(C)]
        struct b2a_myers_match {
            ambig: *const u8,
            wildcards: *const u8,
        }
        #[link(name = "b200align")]
        extern "C" {
            fn b2a_myers_batch(e: *mut c_void, m: *const b2a_myers_match, k: u32, pairs: *const b2a_pairs,
                               best_end: *mut u32, best_dist: *mut u32, n_hits: *mut u64, status: *mut u32,
                               stats: *mut c_void) -> i32;
            fn b2a_myers_hits_fetch(e: *mut c_void, hit_off: *mut u64, hit_end: *mut u32, hit_dist: *mut u32) -> i32;
        }

        /// The bit-vector types of the simple variant: `Myers<u64>` takes patterns of up to 64 symbols, `Myers<u128>`
        /// up to 128 (simple.rs:49-53); for `long::Myers` they only set the initial max_dist (long.rs:583-590).
        pub trait BitVec {
            const BITS: usize;
        }
        impl BitVec for u64 {
            const BITS: usize = 64;
        }
        impl BitVec for u128 {
            const BITS: usize = 128;
        }

        /// A pattern with its match relation (builder.rs): ambiguity rows (bit t of row p: pattern byte p also
        /// matches text byte t) and text wildcards, in the tables b2a_myers_match takes.
        #[derive(Clone)]
        struct Searcher {
            pattern: Vec<u8>,
            ambig: Option<Vec<u8>>,
            wildcards: Option<Vec<u8>>,
        }

        impl Searcher {
            /// per text: the first end of the least distance (None for an empty text) and, with k, every
            /// (end, distance) with distance <= k in ascending end order
            fn search(&self, texts: &[&[u8]], k: Option<u32>) -> (Vec<Option<(usize, u32)>>, Vec<Vec<(usize, u32)>>) {
                let n = texts.len();
                let mut blob = self.pattern.clone();
                let (mut y_off, mut y_len) = (Vec::with_capacity(n), Vec::with_capacity(n));
                for t in texts {
                    assert!(t.len() < (1usize << 31), "b200align: a text longer than 2^31 - 1");
                    y_off.push(blob.len() as u64);
                    y_len.push(t.len() as u32);
                    blob.extend_from_slice(t);
                }
                let (x_off, x_len) = (vec![0u64; n], vec![self.pattern.len() as u32; n]);
                let cp = b2a_pairs { seq_blob: blob.as_ptr(), x_off: x_off.as_ptr(), x_len: x_len.as_ptr(),
                                     y_off: y_off.as_ptr(), y_len: y_len.as_ptr(), blob_bytes: blob.len() as u64,
                                     n_pairs: n as u64 };
                let cm = b2a_myers_match {
                    ambig: self.ambig.as_ref().map_or(std::ptr::null(), |v| v.as_ptr()),
                    wildcards: self.wildcards.as_ref().map_or(std::ptr::null(), |v| v.as_ptr()),
                };
                let (mut be, mut bd) = (vec![0u32; n], vec![0u32; n]);
                let mut n_hits = 0u64;
                let mut lists = vec![Vec::new(); if k.is_some() { n } else { 0 }];
                if n > 0 {
                    let hits_ptr: *mut u64 = if k.is_some() { &mut n_hits } else { std::ptr::null_mut() };
                    with_engine(|e| unsafe {
                        b2a_myers_batch(e, &cm, k.unwrap_or(0), &cp, be.as_mut_ptr(), bd.as_mut_ptr(), hits_ptr,
                                        std::ptr::null_mut(), std::ptr::null_mut())
                    });
                    if k.is_some() {
                        let mut off = vec![0u64; n + 1];
                        let (mut he, mut hd) = (vec![0u32; n_hits as usize], vec![0u32; n_hits as usize]);
                        with_engine(|e| unsafe { b2a_myers_hits_fetch(e, off.as_mut_ptr(), he.as_mut_ptr(), hd.as_mut_ptr()) });
                        for (i, l) in lists.iter_mut().enumerate() {
                            let (lo, hi) = (off[i] as usize, off[i + 1] as usize);
                            *l = he[lo..hi].iter().zip(&hd[lo..hi]).map(|(&e, &d)| (e as usize, d)).collect();
                        }
                    }
                }
                let best = be.iter().zip(&bd).zip(texts)
                    .map(|((&e, &d), t)| if t.is_empty() { None } else { Some((e as usize, d)) }).collect();
                (best, lists)
            }
        }

        /// simple.rs: patterns of at most T::BITS symbols, distances as u8
        pub struct Myers<T: BitVec = u64> {
            s: Searcher,
            _t: PhantomData<T>,
        }

        impl<T: BitVec> Myers<T> {
            pub fn new(pattern: &[u8]) -> Self {
                MyersBuilder::new().build(pattern)
            }

            /// myers_impl.rs:163-181: u8::MAX for an empty text
            pub fn distance_batch(&self, texts: &[&[u8]]) -> Vec<u8> {
                self.s.search(texts, None).0.into_iter().map(|b| b.map_or(u8::MAX, |(_, d)| d as u8)).collect()
            }

            pub fn find_all_end_batch(&self, texts: &[&[u8]], max_dist: u8) -> Vec<Vec<(usize, u8)>> {
                let lists = self.s.search(texts, Some(max_dist as u32)).1;
                lists.into_iter().map(|l| l.into_iter().map(|(e, d)| (e, d as u8)).collect()).collect()
            }

            /// myers_impl.rs:199-207: the first end of the least distance; panics on an empty text (unwrap)
            pub fn find_best_end_batch(&self, texts: &[&[u8]]) -> Vec<(usize, u8)> {
                self.s.search(texts, None).0.into_iter().map(|b| b.map(|(e, d)| (e, d as u8)).unwrap()).collect()
            }

            pub fn distance(&self, text: &[u8]) -> u8 {
                self.distance_batch(&[text])[0]
            }

            pub fn find_all_end(&self, text: &[u8], max_dist: u8) -> Vec<(usize, u8)> {
                self.find_all_end_batch(&[text], max_dist).pop().unwrap()
            }

            pub fn find_best_end(&self, text: &[u8]) -> (usize, u8) {
                self.find_best_end_batch(&[text])[0]
            }
        }

        /// long.rs: patterns of any length, distances as usize
        pub mod long {
            use super::{BitVec, MyersBuilder, Searcher};
            use std::marker::PhantomData;

            pub struct Myers<T: BitVec = u64> {
                pub(super) s: Searcher,
                pub(super) _t: PhantomData<T>,
            }

            impl<T: BitVec> Myers<T> {
                pub fn new(pattern: &[u8]) -> Self {
                    MyersBuilder::new().build_long(pattern)
                }

                fn max_dist() -> usize {
                    usize::MAX - T::BITS  // long.rs:583-590
                }

                pub fn distance_batch(&self, texts: &[&[u8]]) -> Vec<usize> {
                    self.s.search(texts, None).0.into_iter().map(|b| b.map_or(Self::max_dist(), |(_, d)| d as usize)).collect()
                }

                /// max_dist.min(usize::MAX - w); a distance is at most the pattern length (< 2^31), so a bound is
                /// passed on as at most u32::MAX without changing the hits
                pub fn find_all_end_batch(&self, texts: &[&[u8]], max_dist: usize) -> Vec<Vec<(usize, usize)>> {
                    let k = max_dist.min(Self::max_dist()).min(u32::MAX as usize) as u32;
                    let lists = self.s.search(texts, Some(k)).1;
                    lists.into_iter().map(|l| l.into_iter().map(|(e, d)| (e, d as usize)).collect()).collect()
                }

                pub fn find_best_end_batch(&self, texts: &[&[u8]]) -> Vec<(usize, usize)> {
                    self.s.search(texts, None).0.into_iter().map(|b| b.map(|(e, d)| (e, d as usize)).unwrap()).collect()
                }

                pub fn distance(&self, text: &[u8]) -> usize {
                    self.distance_batch(&[text])[0]
                }

                pub fn find_all_end(&self, text: &[u8], max_dist: usize) -> Vec<(usize, usize)> {
                    self.find_all_end_batch(&[text], max_dist).pop().unwrap()
                }

                pub fn find_best_end(&self, text: &[u8]) -> (usize, usize) {
                    self.find_best_end_batch(&[text])[0]
                }
            }
        }

        /// builder.rs: ambiguous pattern symbols and text wildcards
        #[derive(Default, Clone)]
        pub struct MyersBuilder {
            ambigs: HashMap<u8, Vec<u8>>,
            wildcards: Vec<u8>,
        }

        impl MyersBuilder {
            pub fn new() -> MyersBuilder {
                Self::default()
            }

            pub fn ambig(&mut self, byte: u8, equivalents: &[u8]) -> &mut Self {
                self.ambigs.entry(byte).or_default().extend_from_slice(equivalents);
                self
            }

            pub fn text_wildcard(&mut self, wildcard: u8) -> &mut Self {
                self.wildcards.push(wildcard);
                self
            }

            fn searcher(&self, pattern: &[u8]) -> Searcher {
                let ambig = if self.ambigs.is_empty() { None } else {
                    let mut t = vec![0u8; 256 * 32];
                    for (&p, eqs) in &self.ambigs {
                        for &q in eqs {
                            t[32 * p as usize + (q >> 3) as usize] |= 1 << (q & 7);
                        }
                    }
                    Some(t)
                };
                let wildcards = if self.wildcards.is_empty() { None } else {
                    let mut t = vec![0u8; 32];
                    for &q in &self.wildcards {
                        t[(q >> 3) as usize] |= 1 << (q & 7);
                    }
                    Some(t)
                };
                Searcher { pattern: pattern.to_vec(), ambig, wildcards }
            }

            /// simple.rs:49-53
            pub fn build<T: BitVec>(&self, pattern: &[u8]) -> Myers<T> {
                assert!(pattern.len() <= T::BITS, "Pattern too long");
                assert!(!pattern.is_empty(), "Pattern is empty");
                Myers { s: self.searcher(pattern), _t: PhantomData }
            }

            pub fn build_64(&self, pattern: &[u8]) -> Myers<u64> {
                self.build(pattern)
            }

            pub fn build_128(&self, pattern: &[u8]) -> Myers<u128> {
                self.build(pattern)
            }

            /// long.rs:83-84
            pub fn build_long<T: BitVec>(&self, pattern: &[u8]) -> long::Myers<T> {
                assert!(!pattern.is_empty(), "Pattern is empty");
                assert!(pattern.len() <= usize::MAX / 2, "Pattern too long");
                long::Myers { s: self.searcher(pattern), _t: PhantomData }
            }

            pub fn build_long_64(&self, pattern: &[u8]) -> long::Myers<u64> {
                self.build_long(pattern)
            }

            pub fn build_long_128(&self, pattern: &[u8]) -> long::Myers<u128> {
                self.build_long(pattern)
            }
        }
    }
}

// ---------------------------------------------------------------- stats, reference src/stats
/// `bio::stats` on the GPU: the pair HMM (`pairhmm`).
pub mod stats {
    /// `bio::stats::pairhmm::PairHMM` (reference src/stats/pairhmm/pairhmm.rs): `prob_related` (a batch of one) and
    /// `prob_related_batch` over many emissions sharing one set of tables, on the thread's engine of
    /// `alignment::distance`.  Emissions come as per-base classes (`ClassEmission`); log probabilities are plain
    /// `f64` natural logs (`LogProb`'s inner value).  Where the reference asserts (`PairHMM::new`'s
    /// `ln_one_minus_exp`, a NaN result) this shim panics with the engine's message.
    pub mod pairhmm {
        use std::os::raw::c_void;

        use crate::alignment::distance::with_engine;

        #[repr(C)]
        struct b2a_pairs {
            seq_blob: *const u8,
            x_off: *const u64,
            x_len: *const u32,
            y_off: *const u64,
            y_len: *const u32,
            blob_bytes: u64,
            n_pairs: u64,
        }
        #[repr(C)]
        struct b2a_pairhmm_params {
            prob_gap_x: f64,
            prob_gap_y: f64,
            prob_gap_x_extend: f64,
            prob_gap_y_extend: f64,
            free_start_gap_x: i32,
            free_end_gap_x: i32,
            max_edit_dist: u64,
            n_classes: u32,
            emit_match: *const f64,
            emit_mismatch: *const f64,
            emit_x: *const f64,
            emit_y: *const f64,
            class_blob: *const u8,
        }
        #[link(name = "b200align")]
        extern "C" {
            fn b2a_pairhmm_batch(e: *mut c_void, params: *const b2a_pairhmm_params, pairs: *const b2a_pairs,
                                 prob: *mut f64, status: *mut u32, stats: *mut c_void) -> i32;
        }

        /// GapParameters (mod.rs:140-153), natural logs
        pub trait GapParameters {
            fn prob_gap_x(&self) -> f64;
            fn prob_gap_y(&self) -> f64;
            fn prob_gap_x_extend(&self) -> f64;
            fn prob_gap_y_extend(&self) -> f64;
        }

        /// StartEndGapParameters (mod.rs:155-179); prob_start_gap_x is the trait's default
        pub trait StartEndGapParameters {
            fn free_start_gap_x(&self) -> bool;
            fn free_end_gap_x(&self) -> bool;
        }

        /// Per-base emission classes: `tables` = (emit_match, emit_mismatch, emit_x, emit_y), one natural-log value
        /// per class (1 to 256 classes); `x_classes` / `y_classes` one class byte per base, or None for class 0.
        pub struct ClassEmission<'a> {
            pub x: &'a [u8],
            pub y: &'a [u8],
            pub tables: [&'a [f64]; 4],
            pub x_classes: Option<&'a [u8]>,
            pub y_classes: Option<&'a [u8]>,
        }

        pub struct PairHMM {
            gap: [f64; 4],
        }

        impl PairHMM {
            pub fn new<G: GapParameters>(gap_params: &G) -> Self {
                PairHMM {
                    gap: [gap_params.prob_gap_x(), gap_params.prob_gap_y(), gap_params.prob_gap_x_extend(),
                          gap_params.prob_gap_y_extend()],
                }
            }

            pub fn prob_related<A: StartEndGapParameters>(&mut self, emission: &ClassEmission, alignment_mode: &A,
                                                          max_edit_dist: Option<usize>) -> f64 {
                self.prob_related_batch(std::slice::from_ref(emission), alignment_mode, max_edit_dist)[0]
            }

            pub fn prob_related_batch<A: StartEndGapParameters>(&mut self, emissions: &[ClassEmission],
                                                                alignment_mode: &A, max_edit_dist: Option<usize>)
                                                                -> Vec<f64> {
                let n = emissions.len();
                let mut out = vec![0f64; n];
                if n == 0 {
                    return out;
                }
                let tables = emissions[0].tables;
                let n_classes = tables[0].len();
                assert!((1..=256).contains(&n_classes) && tables.iter().all(|t| t.len() == n_classes),
                        "b200align: four emission tables of 1 .. 256 classes");
                let (mut blob, mut cls) = (Vec::new(), Vec::new());
                let (mut x_off, mut y_off, mut x_len, mut y_len) = (Vec::new(), Vec::new(), Vec::new(), Vec::new());
                let with_classes = emissions.iter().any(|e| e.x_classes.is_some() || e.y_classes.is_some());
                for e in emissions {
                    assert!(e.tables.iter().zip(tables.iter()).all(|(a, b)| a.as_ptr() == b.as_ptr() || a == b),
                            "b200align: every emission of a batch shares one set of tables");
                    assert!(e.x.len() < (1usize << 31) && e.y.len() < (1usize << 31),
                            "b200align: a sequence longer than 2^31 - 1");
                    for (seq, c, off, len) in [(e.x, e.x_classes, &mut x_off, &mut x_len),
                                               (e.y, e.y_classes, &mut y_off, &mut y_len)] {
                        off.push(blob.len() as u64);
                        len.push(seq.len() as u32);
                        blob.extend_from_slice(seq);
                        match c {
                            Some(c) => {
                                assert!(c.len() == seq.len(), "b200align: one class byte per base");
                                cls.extend_from_slice(c)
                            }
                            None => cls.resize(blob.len(), 0),
                        }
                    }
                }
                let params = b2a_pairhmm_params {
                    prob_gap_x: self.gap[0],
                    prob_gap_y: self.gap[1],
                    prob_gap_x_extend: self.gap[2],
                    prob_gap_y_extend: self.gap[3],
                    free_start_gap_x: alignment_mode.free_start_gap_x() as i32,
                    free_end_gap_x: alignment_mode.free_end_gap_x() as i32,
                    max_edit_dist: max_edit_dist.map_or(u64::MAX, |k| k as u64),
                    n_classes: n_classes as u32,
                    emit_match: tables[0].as_ptr(),
                    emit_mismatch: tables[1].as_ptr(),
                    emit_x: tables[2].as_ptr(),
                    emit_y: tables[3].as_ptr(),
                    class_blob: if with_classes { cls.as_ptr() } else { std::ptr::null() },
                };
                let cp = b2a_pairs {
                    seq_blob: blob.as_ptr(),
                    x_off: x_off.as_ptr(),
                    x_len: x_len.as_ptr(),
                    y_off: y_off.as_ptr(),
                    y_len: y_len.as_ptr(),
                    blob_bytes: blob.len() as u64,
                    n_pairs: n as u64,
                };
                // no status array: a NaN result (the reference's assert) fails the call, and with_engine panics
                with_engine(|e| unsafe {
                    b2a_pairhmm_batch(e, &params, &cp, out.as_mut_ptr(), std::ptr::null_mut(), std::ptr::null_mut())
                });
                out
            }
        }
    }
}
