//! GpuMetrics — one object that plays both of the reference's handlers over libkta_gpu.so (include/kta.h).
//! UNCOMPILED / UNTESTED: written against rdkafka 0.25.0 + the reference at 5666ec1; no Rust toolchain exists in
//! the image this repository is built in.
//!
//! main.rs changes (src/main.rs line numbers of the reference):
//!   :77-82   replace `log_compaction_metrics` + `metrics` by
//!            `let mut metrics = GpuMetrics::new(<partition count>, matches.occurrences_of("count-alive-keys") == 1);`
//!            (the partition count is known after get_topic_offsets, :94 — construct there)
//!   :108-115 `topic_analyzer.add_metric_handler(&mut metrics);`   (once)
//!   :117     after read_topic_into_metrics: `metrics.finish();`
//!   :130-170 the getters below have the reference's names; `l.sum_all_alive()` becomes `metrics.sum_all_alive()`.
use kafka::MetricHandler;
use rdkafka::message::{BorrowedMessage, Message};
use std::os::raw::{c_char, c_int};

#[repr(C)]
pub struct KtaConfig {
    struct_size: i32, device: i32, num_partitions: i32, count_alive_keys: i32, hll_precision: i32, alive_table_kib: i32,
    ring_records: i64, ring_key_bytes: i64, now_s: i64, now_ns: i32, isolation_level: i32, shard_world: i32, shard_rank: i32,
}
#[repr(C)]
pub struct KtaHandle { _private: [u8; 0] }

extern "C" {
    fn kta_create(cfg: *const KtaConfig, out: *mut *mut KtaHandle) -> c_int;
    fn kta_destroy(h: *mut KtaHandle) -> c_int;
    fn kta_push(h: *mut KtaHandle, partition: i32, offset: i64, ts_ms: i64, key: *const u8, key_len: i32, value_len: i32) -> c_int;
    fn kta_finalize(h: *mut KtaHandle) -> c_int;
    fn kta_counter(h: *const KtaHandle, which: c_int, partition: i32, out: *mut u64) -> c_int;
    fn kta_avg(h: *const KtaHandle, which: c_int, partition: i32, out: *mut u64) -> c_int;
    fn kta_dirty_ratio(h: *const KtaHandle, partition: i32, out: *mut f32) -> c_int;
    fn kta_global(h: *const KtaHandle, which: c_int, out: *mut u64) -> c_int;
    fn kta_timestamps(h: *const KtaHandle, earliest_s: *mut i64, earliest_ns: *mut i32, latest_s: *mut i64) -> c_int;
    fn kta_alive_keys(h: *const KtaHandle, out: *mut u64) -> c_int;
    fn kta_last_error() -> *const c_char;
}

const KTA_ERR_DIV_BY_ZERO: c_int = 5;

pub struct GpuMetrics { h: *mut KtaHandle }

fn last_error() -> String {
    unsafe { std::ffi::CStr::from_ptr(kta_last_error()) }.to_string_lossy().into_owned()
}

impl GpuMetrics {
    pub fn new(num_partitions: i32, count_alive_keys: bool) -> GpuMetrics {
        let cfg = KtaConfig {
            struct_size: std::mem::size_of::<KtaConfig>() as i32, device: -1, num_partitions,
            count_alive_keys: count_alive_keys as i32, hll_precision: 0, alive_table_kib: 0, ring_records: 0, ring_key_bytes: 0,
            now_s: i64::MIN, // the library reads the clock itself: earliest_message starts at Utc::now() (metric.rs:39)
            now_ns: 0, isolation_level: 0, shard_world: 0, shard_rank: 0,
        };
        let mut h = std::ptr::null_mut();
        if unsafe { kta_create(&cfg, &mut h) } != 0 { panic!("kta_create failed: {}", last_error()); }
        GpuMetrics { h }
    }
    /// drain the landing ring, wait for the GPU, bring the state to the host; call once after the poll loop
    pub fn finish(&mut self) { if unsafe { kta_finalize(self.h) } != 0 { panic!("kta_finalize failed: {}", last_error()); } }

    fn counter(&self, which: c_int, p: i32) -> u64 { let mut v = 0; unsafe { kta_counter(self.h, which, p, &mut v) }; v }
    fn avg(&self, which: c_int, p: i32) -> u64 {
        let mut v = 0;
        match unsafe { kta_avg(self.h, which, p, &mut v) } {
            0 => v,
            KTA_ERR_DIV_BY_ZERO => panic!("attempt to divide by zero"), // what metric.rs:135,144,153 does
            _ => panic!("kta_avg failed: {}", last_error()),
        }
    }
    fn global(&self, which: c_int) -> u64 { let mut v = 0; unsafe { kta_global(self.h, which, &mut v) }; v }

    pub fn total(&self, p: i32) -> u64 { self.counter(0, p) }
    pub fn tombstones(&self, p: i32) -> u64 { self.counter(1, p) }
    pub fn alive(&self, p: i32) -> u64 { self.counter(2, p) }
    pub fn key_null(&self, p: i32) -> u64 { self.counter(3, p) }
    pub fn key_non_null(&self, p: i32) -> u64 { self.counter(4, p) }
    pub fn key_size_sum(&self, p: i32) -> u64 { self.counter(5, p) }
    pub fn value_size_sum(&self, p: i32) -> u64 { self.counter(6, p) }
    pub fn key_size_avg(&self, p: i32) -> u64 { self.avg(0, p) }
    pub fn value_size_avg(&self, p: i32) -> u64 { self.avg(1, p) }
    pub fn message_size_avg(&self, p: i32) -> u64 { self.avg(2, p) }
    pub fn dirty_ratio(&self, p: i32) -> f32 { let mut v = 0f32; unsafe { kta_dirty_ratio(self.h, p, &mut v) }; v }
    pub fn smallest_message(&self) -> u64 { self.global(0) }
    pub fn largest_message(&self) -> u64 { self.global(1) }
    pub fn overall_size(&self) -> u64 { self.global(2) }
    pub fn overall_count(&self) -> u64 { self.global(3) }
    /// (seconds, nanoseconds) since the epoch; build the chrono values the report prints from these
    pub fn earliest_message(&self) -> (i64, i32) {
        let (mut s, mut ns, mut l) = (0i64, 0i32, 0i64);
        unsafe { kta_timestamps(self.h, &mut s, &mut ns, &mut l) };
        (s, ns)
    }
    pub fn latest_message(&self) -> i64 {
        let (mut s, mut ns, mut l) = (0i64, 0i32, 0i64);
        unsafe { kta_timestamps(self.h, &mut s, &mut ns, &mut l) };
        l
    }
    pub fn sum_all_alive(&self) -> usize { let mut v = 0; unsafe { kta_alive_keys(self.h, &mut v) }; v as usize }
}

impl MetricHandler for GpuMetrics {
    fn handle_message<'b>(&mut self, m: &BorrowedMessage<'b>) where BorrowedMessage<'b>: Message {
        // the accessors the reference's handlers read: src/metric.rs:208-209, 218, 233, 291, 293
        let ts = m.timestamp().to_millis().unwrap_or(-1); // None ⇒ -1 ⇒ treated as 0 by the library (metric.rs:209)
        let (kp, kl) = match m.key() { Some(k) => (k.as_ptr(), k.len() as i32), None => (std::ptr::null(), -1) };
        let vl = match m.payload() { Some(v) => v.len() as i32, None => -1 };
        if unsafe { kta_push(self.h, m.partition(), m.offset(), ts, kp, kl, vl) } != 0 {
            panic!("kta_push failed: {}", last_error());
        }
    }
}

impl Drop for GpuMetrics { fn drop(&mut self) { unsafe { kta_destroy(self.h); } } }
