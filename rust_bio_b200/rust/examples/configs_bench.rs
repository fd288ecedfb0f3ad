//! BASELINE configs C1-C5 timed on rust-bio itself (`bio = "4.0.1"`, CPU) and -- with `--features b200` -- on
//! this crate's `*_batch` methods (libb200align.so), with the same splitmix64 generator as
//! `rust_bio_b200/synth.py` (SURVEY 8d) so both sides and the Python/C++ harness see identical sequences.
//!
//! NOT COMPILED BY THIS REPOSITORY'S BUILD (it needs no Rust toolchain): it ships so that the real crate can be
//! timed wherever one exists.  Workload shape follows rust-bio's own benches/pairwise.rs:140-159
//! (`Aligner::with_capacity(..).local/global/semiglobal`, score 1/-1, gap_open -5, gap_extend -1).
//!
//!   cargo run --release --example configs_bench -- C2 20000 16      # config, pairs (subsample), CPU threads
//!   cargo run --release --features b200 --example configs_bench -- C2 1000000 16
//!
//! Prints one JSON line per arm: {"config","pairs","threads","seconds","gcups","checksum"}; `checksum` is the
//! wrapping sum of all scores (compare it with `python -m tools.config_checksum`).
use bio::alignment::pairwise::{banded, Aligner, Scoring};
use bio::scores::blosum62;
use std::time::Instant;

const GOLDEN: u64 = 0x9E37_79B9_7F4A_7C15;

fn mix(mut z: u64) -> u64 {
    z = (z ^ (z >> 30)).wrapping_mul(0xBF58_476D_1CE4_E5B9);
    z = (z ^ (z >> 27)).wrapping_mul(0x94D0_49BB_1331_11EB);
    z ^ (z >> 31)
}

/// draw k (1-based) of the stream seeded with `seed`: state = seed + k * GOLDEN
fn draw(seed: u64, k: u64) -> u64 {
    mix(seed.wrapping_add(k.wrapping_mul(GOLDEN)))
}

fn random_seq(seed: u64, len: usize, alphabet: &[u8]) -> Vec<u8> {
    (1..=len as u64).map(|k| alphabet[((draw(seed, k) >> 32) % alphabet.len() as u64) as usize]).collect()
}

/// synth.mutated_window_pairs: y uniform (seed BASE+2p+1); x = window of y with 5 % substitutions, 0.5 %
/// insertions, 0.5 % deletions, cut to m symbols.  Draw 0 = window start, draws 1..L = event per source position,
/// draws L+1..2L = the inserted / substituted symbol.
fn mutated_window(base: u64, p: u64, m: usize, n: usize, alphabet: &[u8]) -> (Vec<u8>, Vec<u8>) {
    let a = alphabet.len() as u64;
    let l = m + std::cmp::max(32, m / 8);
    let y = random_seq(base.wrapping_add(2 * p + 1), n, alphabet);
    let sx = base.wrapping_add(2 * p);
    let z = |k: u64| draw(sx, k + 1); // numpy column k of draws(seed, 2L+1)
    let start = ((z(0) >> 32) % (n - l + 1) as u64) as usize;
    let code = |c: u8| alphabet.iter().position(|&q| q == c).unwrap() as u64;
    let mut x = Vec::with_capacity(m + 2);
    for s in 0..l {
        if x.len() >= m {
            break;
        }
        let u = ((z(1 + s as u64) >> 11) as f64) * (1.0 / (1u64 << 53) as f64);
        let r = (z(1 + l as u64 + s as u64) >> 32) % a;
        let src = y[start + s];
        if u < 0.05 {
            x.push(alphabet[((code(src) + 1 + r % (a - 1)) % a) as usize]);
        } else if u < 0.055 {
            x.push(alphabet[r as usize]);
            if x.len() < m {
                x.push(src);
            }
        } else if u < 0.06 {
            // deletion: the source symbol is skipped
        } else {
            x.push(src);
        }
    }
    while x.len() < m {
        x.push(alphabet[0]);
    }
    x.truncate(m);
    (x, y)
}

struct Cfg {
    name: &'static str,
    base: u64,
    m: usize,
    n: usize,
    alphabet: &'static [u8],
    mode: &'static str,
}

const CONFIGS: &[Cfg] = &[
    Cfg { name: "C1", base: 0xB200_0001, m: 150, n: 150, alphabet: b"ACGT", mode: "local" },
    Cfg { name: "C2", base: 0xB200_0002, m: 150, n: 150, alphabet: b"ACGT", mode: "local" },
    Cfg { name: "C3", base: 0xB200_0003, m: 1000, n: 1000, alphabet: b"ACGT", mode: "global" },
    Cfg { name: "C4", base: 0xB200_0004, m: 500, n: 10000, alphabet: b"ACGT", mode: "banded_semiglobal" },
    Cfg { name: "C5", base: 0xB200_0005, m: 10000, n: 10000, alphabet: b"ACDEFGHIKLMNPQRSTVWY", mode: "local_blosum62" },
];

fn pairs_of(c: &Cfg, n_pairs: usize) -> Vec<(Vec<u8>, Vec<u8>)> {
    (0..n_pairs as u64)
        .map(|p| {
            if c.name == "C4" {
                mutated_window(c.base, p, c.m, c.n, c.alphabet)
            } else {
                (random_seq(c.base.wrapping_add(2 * p), c.m, c.alphabet), random_seq(c.base.wrapping_add(2 * p + 1), c.n, c.alphabet))
            }
        })
        .collect()
}

/// rust-bio on `threads` host threads: static partition, one Aligner per thread reused across pairs (mod.rs:505-506)
fn cpu_arm(c: &Cfg, pairs: &[(Vec<u8>, Vec<u8>)], threads: usize) -> (f64, i64, u64) {
    let t0 = Instant::now();
    let chunk = (pairs.len() + threads - 1) / threads;
    let results: Vec<(i64, u64)> = std::thread::scope(|s| {
        let hs: Vec<_> = pairs
            .chunks(chunk.max(1))
            .map(|part| {
                s.spawn(move || {
                    let score = |a: u8, b: u8| if a == b { 1i32 } else { -1i32 };
                    let mut sum = 0i64;
                    let mut cells = 0u64;
                    match c.mode {
                        "local" | "global" => {
                            let mut al = Aligner::with_capacity(c.m, c.n, -5, -1, &score);
                            for (x, y) in part {
                                let a = if c.mode == "local" { al.local(x, y) } else { al.global(x, y) };
                                sum = sum.wrapping_add(a.score as i64);
                                cells += (x.len() * y.len()) as u64;
                            }
                        }
                        "local_blosum62" => {
                            let mut al = Aligner::with_capacity(c.m, c.n, -10, -1, &blosum62);
                            for (x, y) in part {
                                sum = sum.wrapping_add(al.local(x, y).score as i64);
                                cells += (x.len() * y.len()) as u64;
                            }
                        }
                        _ => {
                            let sc = Scoring::from_scores(-5, -1, 1, -1);
                            let mut al = banded::Aligner::with_scoring(sc, 32, 32);
                            for (x, y) in part {
                                sum = sum.wrapping_add(al.semiglobal(x, y).score as i64);
                                cells += (x.len() * y.len()) as u64; // m*n-equivalent; Band::num_cells is private
                            }
                        }
                    }
                    (sum, cells)
                })
            })
            .collect();
        hs.into_iter().map(|h| h.join().unwrap()).collect()
    });
    let secs = t0.elapsed().as_secs_f64();
    (secs, results.iter().fold(0i64, |a, r| a.wrapping_add(r.0)), results.iter().map(|r| r.1).sum())
}

#[cfg(feature = "b200")]
fn gpu_arm(c: &Cfg, pairs: &[(Vec<u8>, Vec<u8>)]) -> (f64, i64) {
    use bio_b200::alignment::pairwise as b2;
    let refs: Vec<(&[u8], &[u8])> = pairs.iter().map(|(x, y)| (x.as_slice(), y.as_slice())).collect();
    let score = |a: u8, b: u8| if a == b { 1i32 } else { -1i32 };
    let t0 = Instant::now();
    let alns = match c.mode {
        "local" => b2::Aligner::with_capacity(c.m, c.n, -5, -1, &score).local_batch(&refs),
        "global" => b2::Aligner::with_capacity(c.m, c.n, -5, -1, &score).global_batch(&refs),
        "local_blosum62" => b2::Aligner::with_capacity(c.m, c.n, -10, -1, &blosum62).local_batch(&refs),
        _ => b2::banded::Aligner::with_scoring(b2::Scoring::from_scores(-5, -1, 1, -1), 32, 32).semiglobal_batch(&refs),
    };
    (t0.elapsed().as_secs_f64(), alns.iter().fold(0i64, |a, r| a.wrapping_add(r.score as i64)))
}

fn main() {
    let args: Vec<String> = std::env::args().collect();
    let name = args.get(1).map(|s| s.as_str()).unwrap_or("C1");
    let c = CONFIGS.iter().find(|c| c.name == name).expect("config must be one of C1..C5");
    let n_pairs: usize = args.get(2).and_then(|s| s.parse().ok()).unwrap_or(1000);
    let threads: usize = args.get(3).and_then(|s| s.parse().ok()).unwrap_or(1);
    let pairs = pairs_of(c, n_pairs);
    let (secs, sum, cells) = cpu_arm(c, &pairs, threads);
    println!(
        "{{\"arm\":\"rust-bio 4.0.1 (CPU)\",\"config\":\"{}\",\"pairs\":{},\"threads\":{},\"seconds\":{:.4},\"gcups\":{:.4},\"checksum\":{}}}",
        c.name, n_pairs, threads, secs, cells as f64 / secs / 1e9, sum
    );
    #[cfg(feature = "b200")]
    {
        let (gs, gsum) = gpu_arm(c, &pairs);
        println!(
            "{{\"arm\":\"bio_b200 (libb200align.so, host in -> host out)\",\"config\":\"{}\",\"pairs\":{},\"seconds\":{:.4},\"gcups\":{:.4},\"checksum\":{},\"checksum_matches_cpu\":{}}}",
            c.name, n_pairs, gs, cells as f64 / gs / 1e9, gsum, gsum == sum
        );
    }
}
