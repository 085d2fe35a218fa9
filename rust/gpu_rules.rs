//! gpu_rules.rs — `impl FixedRule` for the graph algorithms of the hot path over libcozo_gpu.so.
//!
//! Destination: cozo-core/src/fixed_rule/algos/gpu.rs, compiled under `#[cfg(feature = "gpu-b200")]`
//! and registered in DEFAULT_FIXED_RULES (fixed_rule/mod.rs:611-739) under the stock names, so a
//! CozoScript query is unchanged.  Not compiled in the build image (no Rust toolchain); the
//! executable twin with the same control flow is cozo_b200/host/fixed_rule.hpp, which the GPU
//! tests drive.
//!
//! What stays host-side, exactly as in the reference: option parsing (FixedRulePayload getters),
//! the tuple scan with its arity / weight checks, the memcmp encoding of the node keys, and
//! the emission of result tuples into RegularTempStore.  What moves: dense id assignment
//! (fixed_rule/mod.rs:164-179), CSR construction and the algorithm itself.

use std::collections::{BTreeMap, BTreeSet};
use std::os::raw::c_int;
use std::ptr;
use std::sync::atomic::Ordering;

use miette::{bail, miette, Result};
use smartstring::{LazyCompact, SmartString};

use crate::data::expr::Expr;
use crate::data::memcmp::MemCmpEncoder;
use crate::data::symb::Symbol;
use crate::data::value::DataValue;
use crate::fixed_rule::{FixedRule, FixedRuleInputRelation, FixedRulePayload};
use crate::gpu::sys::*;
use crate::parse::SourceSpan;
use crate::runtime::db::Poison;
use crate::runtime::temp_store::RegularTempStore;

/// Result of the one `cozo_gpu_init` of this process.  There is NO CPU fallback on this path (BASELINE
/// north star, INTEGRATION.md §1): a build with the `gpu-b200` feature registers the GPU rules
/// unconditionally, and if the device cannot be initialised every `run` surfaces this error.
static DEVICE: std::sync::OnceLock<std::result::Result<(), String>> = std::sync::OnceLock::new();

pub(crate) fn ensure_device() -> Result<()> {
    let r = DEVICE.get_or_init(|| {
        let device = std::env::var("COZO_GPU_DEVICE").ok().and_then(|s| s.parse().ok()).unwrap_or(0);
        if unsafe { cozo_gpu_init(device) } == COZO_GPU_OK {
            Ok(())
        } else {
            let msg = unsafe { std::ffi::CStr::from_ptr(cozo_gpu_last_error()) };
            Err(msg.to_string_lossy().into_owned())
        }
    });
    match r {
        Ok(()) => Ok(()),
        Err(e) => Err(miette!("gpu-b200: no usable sm_90 device ({}); this build has no CPU path for this rule", e)),
    }
}

/// Map a C-ABI return code to the error the reference raises on the same condition.
fn check(rc: c_int) -> Result<()> {
    match rc {
        COZO_GPU_OK => Ok(()),
        // the caller re-raises the reference's own ProcessKilled (private to Poison::check,
        // runtime/db.rs:1931-1941) through `PoisonMirror::guard`
        COZO_GPU_EKILLED => Err(miette!("Running query is killed before completion")),
        _ => {
            let msg = unsafe { std::ffi::CStr::from_ptr(cozo_gpu_last_error()) };
            Err(miette!("gpu-b200: {}", msg.to_string_lossy()))
        }
    }
}

/// `Poison` is `Arc<AtomicBool>` (runtime/db.rs:1930); the library polls a `const volatile int*`
/// between kernel launches.  AtomicBool is one byte, so the rule mirrors it into an i32 the
/// library can read: sampled once before the FFI call (`ptr`) and then by a 1 ms watcher thread
/// for the duration of the call.
struct PoisonMirror {
    flag: Box<std::sync::atomic::AtomicI32>,
    src: Poison,
    stop: std::sync::Arc<std::sync::atomic::AtomicBool>,
    th: Option<std::thread::JoinHandle<()>>,
}

impl PoisonMirror {
    fn new(src: Poison) -> Self {
        let flag = Box::new(std::sync::atomic::AtomicI32::new(0));
        let stop = std::sync::Arc::new(std::sync::atomic::AtomicBool::new(false));
        let p = &*flag as *const std::sync::atomic::AtomicI32 as usize;
        let (s2, stop2) = (src.clone(), stop.clone());
        // 1 ms poll: the same latency class as the reference's per-iteration poison.check()
        let th = std::thread::spawn(move || {
            let f = unsafe { &*(p as *const std::sync::atomic::AtomicI32) };
            while !stop2.load(Ordering::Relaxed) {
                if s2.0.load(Ordering::Relaxed) {
                    f.store(1, Ordering::Relaxed);
                    return;
                }
                std::thread::sleep(std::time::Duration::from_millis(1));
            }
        });
        Self { flag, src, stop, th: Some(th) }
    }
    /// Run an FFI call; if it reports EKILLED, surface `Poison::check()`'s own error.
    fn guard(&self, rc: c_int) -> Result<()> {
        if rc == COZO_GPU_EKILLED {
            self.src.check()?;
        }
        check(rc)
    }
    fn ptr(&self) -> *const c_int {
        if self.src.0.load(Ordering::Relaxed) {
            self.flag.store(1, Ordering::Relaxed);
        }
        self.flag.as_ptr() as *const c_int
    }
}

impl Drop for PoisonMirror {
    fn drop(&mut self) {
        self.stop.store(true, Ordering::Relaxed);
        if let Some(t) = self.th.take() {
            let _ = t.join();
        }
    }
}

/// An input relation staged on the device as a graph — `as_directed_graph` /
/// `as_directed_weighted_graph` (fixed_rule/mod.rs:136-328).  The host scans the tuples, checks
/// arity and weights with the reference's error precedence, and memcmp-encodes every endpoint key
/// (data/memcmp.rs: equal bytes <=> equal values); the device assigns the dense ids in first-appearance
/// order, `from` before `to`, and builds the CSR (cozo_gpu_graph_stage_keys, graph.cu).  So
/// `indices` is identical to the reference's and no BTreeMap is built.
pub(crate) struct EdgeList {
    pub g: DevGraph,
    pub indices: Vec<DataValue>,
    /// after mirroring
    pub n_edges: usize,
}

impl<'a, 'b> FixedRuleInputRelation<'a, 'b> {
    pub(crate) fn as_edge_list(&self, undirected: bool, weighted: bool) -> Result<EdgeList> {
        let mut tuples = vec![];
        let mut key_bytes: Vec<u8> = vec![];
        let mut key_off: Vec<u64> = vec![0];
        let mut w: Vec<f32> = vec![];
        for tuple in self.iter()? {
            let tuple = tuple?;
            if tuple.len() < 2 {
                bail!(crate::fixed_rule::NotAnEdgeError(self.span()));
            }
            let mut wt = 1.0f32;
            if weighted {
                if let Some(d) = tuple.get(2) {
                    // fixed_rule/mod.rs:243-290: non-numeric, non-finite and negative weights are errors
                    match d.get_float() {
                        Some(x) if x.is_finite() && x >= 0. => wt = x as f32,
                        _ => bail!(crate::fixed_rule::BadEdgeWeightError(d.clone(), self.span())),
                    }
                }
            }
            key_bytes.encode_datavalue(&tuple[0]);
            key_off.push(key_bytes.len() as u64);
            key_bytes.encode_datavalue(&tuple[1]);
            key_off.push(key_bytes.len() as u64);
            if weighted {
                w.push(wt);
            }
            tuples.push(tuple);
        }
        ensure_device()?;
        let m = tuples.len() as u64;
        let mut g: *mut CozoGpuGraph = ptr::null_mut();
        let mut n = 0u32;
        check(unsafe {
            cozo_gpu_graph_stage_keys(
                &mut g, m, key_bytes.as_ptr(), key_off.as_ptr(),
                if weighted { w.as_ptr() } else { ptr::null() },
                undirected as i32, &mut n,
            )
        })?;
        let g = DevGraph(g);
        let mut first = vec![0u64; n as usize];
        check(unsafe { cozo_gpu_graph_node_endpoints(g.0, first.as_mut_ptr()) })?;
        // endpoint i is field i % 2 of edge (= tuple) i / 2
        let indices = first.iter().map(|&ep| tuples[(ep / 2) as usize][(ep % 2) as usize].clone()).collect();
        Ok(EdgeList { g, indices, n_edges: if undirected { 2 * m as usize } else { m as usize } })
    }
}

impl EdgeList {
    /// dense id of the first field of every row of `rel` that the graph has (starting / goal nodes)
    fn lookup_first_fields(&self, rel: &FixedRuleInputRelation<'_, '_>) -> Result<Vec<u32>> {
        let mut key_bytes: Vec<u8> = vec![];
        let mut key_off: Vec<u64> = vec![0];
        for t in rel.iter()? {
            key_bytes.encode_datavalue(&t?[0]);
            key_off.push(key_bytes.len() as u64);
        }
        let count = key_off.len() - 1;
        let mut ids = vec![COZO_GPU_NONE; count];
        if count > 0 {
            check(unsafe {
                cozo_gpu_graph_lookup_keys(self.g.0, key_bytes.as_ptr(), key_off.as_ptr(), count as u32, ids.as_mut_ptr())
            })?;
        }
        Ok(ids.into_iter().filter(|&i| i != COZO_GPU_NONE).collect())
    }
    /// the dense edge stream in out-CSR order: by (src, dst), parallel edges in input order
    fn edges(&self) -> Result<(Vec<u32>, Vec<u32>, Vec<f32>)> {
        let n = self.indices.len();
        let mut ptr_ = vec![0u32; n + 1];
        let (mut dst, mut w) = (vec![0u32; self.n_edges], vec![0f32; self.n_edges]);
        check(unsafe {
            cozo_gpu_graph_export(self.g.0, ptr_.as_mut_ptr(), dst.as_mut_ptr(), w.as_mut_ptr(), ptr::null_mut(), ptr::null_mut())
        })?;
        let mut src = vec![0u32; self.n_edges];
        for u in 0..n {
            for e in ptr_[u]..ptr_[u + 1] {
                src[e as usize] = u as u32;
            }
        }
        Ok((src, dst, w))
    }
}

/// RAII handle of a staged graph.
pub(crate) struct DevGraph(*mut CozoGpuGraph);

impl Drop for DevGraph {
    fn drop(&mut self) {
        unsafe { cozo_gpu_graph_free(self.0) }
    }
}

// ---------------------------------------------------------------------------------------------
// PageRank (algos/pagerank.rs:26-56)
// ---------------------------------------------------------------------------------------------
pub(crate) struct PageRankGpu;

impl FixedRule for PageRankGpu {
    fn run(&self, payload: FixedRulePayload<'_, '_>, out: &mut RegularTempStore, poison: Poison) -> Result<()> {
        let edges = payload.get_input(0)?;
        let undirected = payload.bool_option("undirected", Some(false))?;
        let theta = payload.unit_interval_option("theta", Some(0.85))? as f32;
        let epsilon = payload.unit_interval_option("epsilon", Some(0.0001))? as f32;
        let iterations = payload.pos_integer_option("iterations", Some(10))?;

        let el = edges.as_edge_list(undirected, false)?;
        if el.indices.is_empty() {
            return Ok(());
        }
        let g = &el.g;
        let pm = PoisonMirror::new(poison);
        let mut ranks = vec![0f32; el.indices.len()];
        let (mut iters, mut err, mut ms) = (0u32, 0f64, 0f64);
        pm.guard(unsafe {
            cozo_gpu_pagerank(
                g.0, theta, epsilon as f64, iterations as u32,
                ranks.as_mut_ptr(), &mut iters, &mut err, &mut ms, pm.ptr(),
            )
        })?;
        for (idx, score) in ranks.iter().enumerate() {
            out.put(vec![el.indices[idx].clone(), DataValue::from(*score as f64)]);
        }
        Ok(())
    }
    fn arity(&self, _o: &BTreeMap<SmartString<LazyCompact>, Expr>, _h: &[Symbol], _s: SourceSpan) -> Result<usize> {
        Ok(2)
    }
}

// ---------------------------------------------------------------------------------------------
// ShortestPathDijkstra (algos/shortest_path_dijkstra.rs:32-160)
//   without a termination relation: one cozo_gpu_sssp_multi over all starting nodes, one row per node,
//   the path rebuilt from `pred` (keep_ties is only honoured with a termination relation, :85-87).
//   with one: cozo_gpu_sssp_goals, where each search stops once its goals are settled (:312-315) and only
//   the goal answers come back: a path per (start, goal), or with keep_ties the tied-predecessor edges
//   leading back from the goals, walked as dijkstra_keep_ties walks its predecessor lists (:397-426).
// ---------------------------------------------------------------------------------------------
/// `tied`: (v, p) pairs of one source, sorted by v
fn collect_tied_paths(
    tied: &[(u32, u32)], start: u32, chain: &mut Vec<u32>, paths: &mut Vec<Vec<u32>>, poison: &Poison,
) -> Result<()> {
    let last = *chain.last().unwrap();
    let from = tied.partition_point(|&(v, _)| v < last);
    for &(_, p) in tied[from..].iter().take_while(|&&(v, _)| v == last) {
        poison.check()?;
        chain.push(p);
        if p == start {
            paths.push(chain.iter().rev().copied().collect());
        } else {
            collect_tied_paths(tied, start, chain, paths, poison)?;
        }
        chain.pop();
    }
    Ok(())
}

pub(crate) struct ShortestPathDijkstraGpu;

impl FixedRule for ShortestPathDijkstraGpu {
    fn run(&self, payload: FixedRulePayload<'_, '_>, out: &mut RegularTempStore, poison: Poison) -> Result<()> {
        let keep_ties = payload.bool_option("keep_ties", Some(false))?;
        let edges = payload.get_input(0)?;
        let starting = payload.get_input(1)?;
        let termination = payload.get_input(2);
        let undirected = payload.bool_option("undirected", Some(false))?;

        let el = edges.as_edge_list(undirected, true)?;
        let starting_nodes: BTreeSet<u32> = el.lookup_first_fields(&starting)?.into_iter().collect();
        let termination_nodes = match termination {
            Err(_) => None,
            Ok(t) => Some(el.lookup_first_fields(&t)?.into_iter().collect::<BTreeSet<u32>>()),
        };
        if starting_nodes.is_empty() || el.indices.is_empty() {
            return Ok(());
        }
        let n = el.indices.len();
        let sources: Vec<u32> = starting_nodes.iter().copied().collect();
        let g = &el.g;
        let pm = PoisonMirror::new(poison.clone());
        let mut ms = 0f64;
        let row = |out: &mut RegularTempStore, start: u32, target: u32, cost: f32, path: &[u32]| {
            out.put(vec![
                el.indices[start as usize].clone(),
                el.indices[target as usize].clone(),
                DataValue::from(cost as f64),
                DataValue::List(path.iter().map(|&u| el.indices[u as usize].clone()).collect()),
            ]);
        };
        let goals: Vec<u32> = match &termination_nodes {
            None => {
                // Goal for (): one row per node, in node order (:233-235)
                let mut dist = vec![0f32; sources.len() * n];
                let mut pred = vec![0u32; sources.len() * n];
                pm.guard(unsafe {
                    cozo_gpu_sssp_multi(
                        g.0, sources.as_ptr(), sources.len() as u32,
                        dist.as_mut_ptr(), pred.as_mut_ptr(), &mut ms, pm.ptr(),
                    )
                })?;
                for (si, &start) in sources.iter().enumerate() {
                    let (d, p) = (&dist[si * n..(si + 1) * n], &pred[si * n..(si + 1) * n]);
                    for target in 0..n as u32 {
                        let mut path = vec![];
                        if d[target as usize].is_finite() {
                            let mut cur = target;
                            path.push(cur);
                            while cur != start {
                                cur = p[cur as usize];
                                path.push(cur);
                            }
                            path.reverse();
                        }
                        row(out, start, target, d[target as usize], &path);
                    }
                }
                return Ok(());
            }
            Some(tn) => tn.iter().copied().collect(),
        };
        // an empty termination set is already exhausted (Goal for BTreeSet, :260-272): no rows
        if goals.is_empty() {
            return Ok(());
        }
        let (ns, ng) = (sources.len(), goals.len());
        let mut cost = vec![0f32; ns * ng];
        let mut off = vec![0u64; if keep_ties { ns + 1 } else { ns * ng + 1 }];
        let mut rows: Vec<u32>;
        let mut cap = 16 * (ns * ng) as u64; // a first guess; the call reports the total when it does not fit
        loop {
            rows = vec![0u32; (cap.max(1) as usize) * if keep_ties { 2 } else { 1 }];
            let (po, pp, pc, to, te, tc) = if keep_ties {
                (ptr::null_mut(), ptr::null_mut(), 0, off.as_mut_ptr(), rows.as_mut_ptr(), cap)
            } else {
                (off.as_mut_ptr(), rows.as_mut_ptr(), cap, ptr::null_mut(), ptr::null_mut(), 0)
            };
            pm.guard(unsafe {
                cozo_gpu_sssp_goals(
                    g.0, sources.as_ptr(), ns as u32, goals.as_ptr(), ng as u32, keep_ties as i32,
                    cost.as_mut_ptr(), po, pp, pc, to, te, tc, &mut ms, pm.ptr(),
                )
            })?;
            let total = *off.last().unwrap();
            if total <= cap {
                break;
            }
            cap = total;
        }
        for (si, &start) in sources.iter().enumerate() {
            let mut tied: Vec<(u32, u32)> = vec![];
            if keep_ties {
                tied = (off[si]..off[si + 1]).map(|e| (rows[2 * e as usize], rows[2 * e as usize + 1])).collect();
                tied.sort_unstable();
            }
            for (gi, &target) in goals.iter().enumerate() {
                let c = cost[si * ng + gi];
                if !c.is_finite() {
                    row(out, start, target, c, &[]); // :322-323
                } else if !keep_ties {
                    let (b, e) = (off[si * ng + gi] as usize, off[si * ng + gi + 1] as usize);
                    row(out, start, target, c, &rows[b..e]); // :325-333
                } else if target != start {
                    // no predecessor of the start: the reference emits nothing for it (:410-421)
                    let (mut chain, mut paths) = (vec![target], vec![]);
                    collect_tied_paths(&tied, start, &mut chain, &mut paths, &poison)?;
                    for path in paths {
                        row(out, start, target, c, &path);
                    }
                }
            }
        }
        Ok(())
    }
    fn arity(&self, _o: &BTreeMap<SmartString<LazyCompact>, Expr>, _h: &[Symbol], _s: SourceSpan) -> Result<usize> {
        Ok(4)
    }
}

// ---------------------------------------------------------------------------------------------
// ClosenessCentrality / BetweennessCentrality (algos/all_pairs_shortest_path.rs:29-197)
// ---------------------------------------------------------------------------------------------
macro_rules! centrality_rule {
    ($name:ident, $entry:ident) => {
        pub(crate) struct $name;
        impl FixedRule for $name {
            fn run(&self, payload: FixedRulePayload<'_, '_>, out: &mut RegularTempStore, poison: Poison) -> Result<()> {
                let edges = payload.get_input(0)?;
                let undirected = payload.bool_option("undirected", Some(false))?;
                let el = edges.as_edge_list(undirected, true)?;
                if el.indices.is_empty() {
                    return Ok(());
                }
                let g = &el.g;
                let pm = PoisonMirror::new(poison);
                let mut res = vec![0f32; el.indices.len()];
                let mut ms = 0f64;
                pm.guard(unsafe { $entry(g.0, res.as_mut_ptr(), &mut ms, pm.ptr()) })?;
                for (i, s) in res.into_iter().enumerate() {
                    out.put(vec![el.indices[i].clone(), DataValue::from(s as f64)]);
                }
                Ok(())
            }
            fn arity(&self, _o: &BTreeMap<SmartString<LazyCompact>, Expr>, _h: &[Symbol], _s: SourceSpan) -> Result<usize> {
                Ok(2)
            }
        }
    };
}
centrality_rule!(ClosenessCentralityGpu, cozo_gpu_closeness);
centrality_rule!(BetweennessCentralityGpu, cozo_gpu_betweenness);

// ---------------------------------------------------------------------------------------------
// ClusteringCoefficients (algos/triangles.rs:26-92): rows [node, coefficient, triangles, degree]
// ---------------------------------------------------------------------------------------------
pub(crate) struct ClusteringCoefficientsGpu;

impl FixedRule for ClusteringCoefficientsGpu {
    fn run(&self, payload: FixedRulePayload<'_, '_>, out: &mut RegularTempStore, poison: Poison) -> Result<()> {
        let edges = payload.get_input(0)?;
        // triangles.rs:34: always undirected
        let el = edges.as_edge_list(true, false)?;
        if el.indices.is_empty() {
            return Ok(());
        }
        let n = el.indices.len();
        let g = &el.g;
        let pm = PoisonMirror::new(poison);
        let (mut cc, mut tri, mut deg) = (vec![0f64; n], vec![0u64; n], vec![0u64; n]);
        let mut ms = 0f64;
        pm.guard(unsafe {
            cozo_gpu_clustering(g.0, cc.as_mut_ptr(), tri.as_mut_ptr(), deg.as_mut_ptr(), &mut ms, pm.ptr())
        })?;
        for i in 0..n {
            out.put(vec![
                el.indices[i].clone(),
                DataValue::from(cc[i]),
                DataValue::from(tri[i] as i64),
                DataValue::from(deg[i] as i64),
            ]);
        }
        Ok(())
    }
    fn arity(&self, _o: &BTreeMap<SmartString<LazyCompact>, Expr>, _h: &[Symbol], _s: SourceSpan) -> Result<usize> {
        Ok(4)
    }
}

// ---------------------------------------------------------------------------------------------
// KShortestPathYen (algos/yen.rs:26-211).  The control flow of k_shortest_path_yen stays; the dijkstra
// calls of one round — every spur node of every (start, goal) pair — become ONE batch of goal-directed
// searches with their ForbiddenEdge / ForbiddenNode sets (cozo_gpu_sssp_paths).  Executable twin:
// cozo_b200/host/fixed_rule.hpp `KShortestPathYen` (tested against the oracle).
// ---------------------------------------------------------------------------------------------
pub(crate) struct KShortestPathYenGpu;

struct YenSearch {
    pair: usize,
    i: usize, // spur index; usize::MAX = the initial search
    from: u32,
    forb_nodes: Vec<u32>,
    forb_edges: Vec<(u32, u32)>,
}

fn yen_batch(g: &DevGraph, goals: &[u32], batch: &[YenSearch], pm: &PoisonMirror) -> Result<Vec<(f32, Vec<u32>)>> {
    let k = batch.len();
    if k == 0 {
        return Ok(vec![]);
    }
    let src: Vec<u32> = batch.iter().map(|b| b.from).collect();
    let goal: Vec<u32> = batch.iter().map(|b| goals[b.pair]).collect();
    let (mut fnp, mut fep) = (vec![0u32; k + 1], vec![0u32; k + 1]);
    let (mut fnn, mut fes, mut fed) = (vec![], vec![], vec![]);
    for (b, s) in batch.iter().enumerate() {
        fnn.extend_from_slice(&s.forb_nodes);
        for &(a, c) in &s.forb_edges {
            fes.push(a);
            fed.push(c);
        }
        fnp[b + 1] = fnn.len() as u32;
        fep[b + 1] = fes.len() as u32;
    }
    if fnn.is_empty() {
        fnn.push(0);
    }
    if fes.is_empty() {
        fes.push(0);
        fed.push(0);
    }
    let mut max_len = 64u32;
    loop {
        let (mut cost, mut len) = (vec![0f32; k], vec![0u32; k]);
        let mut paths = vec![0u32; k * max_len as usize];
        let mut ms = 0f64;
        pm.guard(unsafe {
            cozo_gpu_sssp_paths(
                g.0, src.as_ptr(), goal.as_ptr(), k as u32, fnp.as_ptr(), fnn.as_ptr(), fep.as_ptr(), fes.as_ptr(),
                fed.as_ptr(), max_len, cost.as_mut_ptr(), len.as_mut_ptr(), paths.as_mut_ptr(), &mut ms, pm.ptr(),
            )
        })?;
        let need = len.iter().copied().max().unwrap_or(0);
        if need > max_len {
            max_len = need; // a path did not fit: same batch again with a larger buffer
            continue;
        }
        return Ok((0..k)
            .map(|b| (cost[b], paths[b * max_len as usize..b * max_len as usize + len[b] as usize].to_vec()))
            .collect());
    }
}

impl FixedRule for KShortestPathYenGpu {
    fn run(&self, payload: FixedRulePayload<'_, '_>, out: &mut RegularTempStore, poison: Poison) -> Result<()> {
        let edges = payload.get_input(0)?;
        let starting = payload.get_input(1)?;
        let termination = payload.get_input(2)?;
        let undirected = payload.bool_option("undirected", Some(false))?; // yen.rs:38
        let k = payload.pos_integer_option("k", None)?; // yen.rs:39
        let el = edges.as_edge_list(undirected, true)?;
        // yen.rs:43-58
        let starts: BTreeSet<u32> = el.lookup_first_fields(&starting)?.into_iter().collect();
        let goals_set: BTreeSet<u32> = el.lookup_first_fields(&termination)?.into_iter().collect();
        struct Pair {
            start: u32,
            k_shortest: Vec<(f32, Vec<u32>)>,
            candidates: Vec<(f32, Vec<u32>)>,
            done: bool,
        }
        let (mut ps, mut goals) = (vec![], vec![]);
        for &s0 in &starts {
            for &g0 in &goals_set {
                ps.push(Pair { start: s0, k_shortest: vec![], candidates: vec![], done: false });
                goals.push(g0);
            }
        }
        if ps.is_empty() {
            return Ok(());
        }
        // the first edge s->d in adjacency order supplies the root-path cost (yen.rs:171-183); the CSR
        // keeps parallel edges in input order
        let mut first_edge: BTreeMap<(u32, u32), f32> = BTreeMap::new();
        let (src, dst, w) = el.edges()?;
        for e in 0..src.len() {
            first_edge.entry((src[e], dst[e])).or_insert(w[e]);
        }
        let g = &el.g;
        let pm = PoisonMirror::new(poison.clone());
        let batch: Vec<YenSearch> = (0..ps.len())
            .map(|pi| YenSearch { pair: pi, i: usize::MAX, from: ps[pi].start, forb_nodes: vec![], forb_edges: vec![] })
            .collect();
        for (b, r) in yen_batch(&g, &goals, &batch, &pm)?.into_iter().enumerate() {
            ps[batch[b].pair].k_shortest.push(r); // yen.rs:130-136
        }
        for _ in 1..k {
            // yen.rs:138
            let mut batch = vec![];
            for (pi, p) in ps.iter().enumerate() {
                if p.done {
                    continue;
                }
                let prev = &p.k_shortest.last().unwrap().1;
                for i in 0..prev.len().saturating_sub(1) {
                    let mut s = YenSearch { pair: pi, i, from: prev[i], forb_nodes: prev[..i].to_vec(), forb_edges: vec![] };
                    for (_, path) in &p.k_shortest {
                        // yen.rs:147-155
                        if path.len() >= i + 2 && path[..=i] == prev[..=i] {
                            s.forb_edges.push((path[i], path[i + 1]));
                        }
                    }
                    batch.push(s);
                }
            }
            let res = yen_batch(&g, &goals, &batch, &pm)?;
            for (b, (spur_cost, spur_path)) in res.into_iter().enumerate() {
                let p = &mut ps[batch[b].pair];
                let prev = p.k_shortest.last().unwrap().1.clone();
                let i = batch[b].i;
                let mut total = spur_cost;
                for j in 0..i {
                    if let Some(w) = first_edge.get(&(prev[j], prev[j + 1])) {
                        total += *w;
                    }
                }
                let mut total_path = prev[..i].to_vec();
                total_path.extend(spur_path);
                if !p.candidates.iter().any(|c| c.1 == total_path) {
                    p.candidates.push((total, total_path)); // yen.rs:187-189
                }
            }
            poison.check()?;
            for p in ps.iter_mut() {
                if p.done {
                    continue;
                }
                if p.candidates.is_empty() {
                    p.done = true; // yen.rs:194-196
                    continue;
                }
                p.candidates.sort_by(|a, b| b.0.total_cmp(&a.0)); // stable, descending: yen.rs:197
                let shortest = p.candidates.pop().unwrap();
                if shortest.0.is_finite() {
                    p.k_shortest.push(shortest); // yen.rs:200-203
                }
            }
        }
        for (pi, p) in ps.iter().enumerate() {
            for (cost, path) in &p.k_shortest {
                // yen.rs:62-77, 103-117
                out.put(vec![
                    el.indices[p.start as usize].clone(),
                    el.indices[goals[pi] as usize].clone(),
                    DataValue::from(*cost as f64),
                    DataValue::List(path.iter().map(|u| el.indices[*u as usize].clone()).collect()),
                ]);
            }
        }
        Ok(())
    }
    fn arity(&self, _o: &BTreeMap<SmartString<LazyCompact>, Expr>, _h: &[Symbol], _s: SourceSpan) -> Result<usize> {
        Ok(4)
    }
}

/// Called from the `lazy_static! DEFAULT_FIXED_RULES` block (fixed_rule/mod.rs:611-739) after the stock
/// insertions.  A binary built with `--features gpu-b200` runs these rules on the device, full stop: the GPU
/// rules replace the stock entries under the same names unconditionally, and a missing / unusable device is
/// reported by `ensure_device()` as the query's error (INTEGRATION.md §1).  Nothing falls back to the CPU
/// implementations silently.
pub(crate) fn register(rules: &mut BTreeMap<String, std::sync::Arc<Box<dyn FixedRule>>>) {
    use std::sync::Arc;
    rules.insert("PageRank".into(), Arc::new(Box::new(PageRankGpu)));
    rules.insert("ShortestPathDijkstra".into(), Arc::new(Box::new(ShortestPathDijkstraGpu)));
    rules.insert("ClosenessCentrality".into(), Arc::new(Box::new(ClosenessCentralityGpu)));
    rules.insert("BetweennessCentrality".into(), Arc::new(Box::new(BetweennessCentralityGpu)));
    rules.insert("ClusteringCoefficients".into(), Arc::new(Box::new(ClusteringCoefficientsGpu)));
    rules.insert("KShortestPathYen".into(), Arc::new(Box::new(KShortestPathYenGpu)));
}
