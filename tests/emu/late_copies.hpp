// late_copies.hpp — TEST INFRASTRUCTURE ONLY: a stricter model of mbarrier + cp.async.bulk for the CPU SIMT emulator.
// tests/test_prune_stream_cpu.py builds a variant of the emulated library in which this section replaces the one of
// cuda_emu.hpp (between the "---- mbarrier + 1-D bulk copy" banner and fence_proxy_async_smem).  There a bulk copy
// completes LATE, as on the device, so a kernel that reads a slot before its wait, or refills a slot whose copy is still
// outstanding, fails on the CPU instead of trapping on a GPU.
// ---- mbarrier + 1-D bulk copy (what common.cuh implements with PTX) ---------------------------------------------------
// bar = { low 32 bits: pending transaction bytes ; bit 32: phase }
// A bulk copy completes LATE, as on the device: bulk_g2s poisons the destination (0xFF bytes: NaN floats, NONE ids) and
// records the copy; a later poll of its barrier (the 1st to 4th, in an order seeded by COZO_EMU_COPY_SEED and the
// barrier's address) performs it and, once the expected bytes are in, flips the phase.  So reading a slot before its
// wait reads poison, and issuing a copy into a slot whose previous copy is still outstanding, or re-initialising a
// barrier with a copy outstanding, aborts.
namespace emu {
struct PendingCopy {
  void* dst;
  const void* src;
  uint32_t bytes;
  uint32_t polls;  // polls of the barrier left before the copy lands
};
inline std::mutex copy_mu;
inline std::vector<std::pair<uint64_t*, PendingCopy>> copies;  // in issue order
inline uint64_t copy_seq = 0;
inline uint64_t copy_seed() {
  static const uint64_t s = [] {
    const char* e = std::getenv("COZO_EMU_COPY_SEED");
    return e ? std::strtoull(e, nullptr, 0) : 1ull;
  }();
  return s;
}
inline uint32_t copy_delay(const uint64_t* bar) {
  uint64_t x = copy_seed() * 0x9E3779B97F4A7C15ull ^ (uint64_t)(uintptr_t)bar ^ (++copy_seq << 32);
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return 1 + (uint32_t)((x ^ (x >> 31)) & 3);
}
}  // namespace emu

inline void mbar_init(uint64_t* bar, uint32_t) {
  {
    std::lock_guard<std::mutex> lk(emu::copy_mu);
    for (auto& c : emu::copies)
      if (c.first == bar) { std::fprintf(stderr, "emu: mbarrier re-initialised while a bulk copy on it is outstanding\n"); std::abort(); }
  }
  __atomic_store_n(bar, 0ull, __ATOMIC_SEQ_CST);
}
inline void mbar_fence_init() {}
inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { __atomic_fetch_add(bar, (uint64_t)bytes, __ATOMIC_SEQ_CST); }
inline bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  {
    std::lock_guard<std::mutex> lk(emu::copy_mu);
    for (size_t i = 0; i < emu::copies.size();) {
      auto& [b, c] = emu::copies[i];
      if (b != bar || --c.polls > 0) { ++i; continue; }
      std::memcpy(c.dst, c.src, c.bytes);
      const uint64_t left = __atomic_sub_fetch(bar, (uint64_t)c.bytes, __ATOMIC_SEQ_CST) & 0xFFFFFFFFull;
      if (left == 0) __atomic_fetch_xor(bar, 1ull << 32, __ATOMIC_SEQ_CST);  // all expected bytes have landed
      emu::copies.erase(emu::copies.begin() + (std::ptrdiff_t)i);
    }
  }
  return ((__atomic_load_n(bar, __ATOMIC_SEQ_CST) >> 32) & 1ull) != parity;
}
inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  unsigned long spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    emu::lane_yield();  // the lane that issues the copy may be a sibling that has not run yet
    if (++spins > (1ul << 28)) __trap();
  }
}
inline void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  if (((uintptr_t)gmem_src & 15) || (bytes & 15)) { std::fprintf(stderr, "emu: cp.async.bulk needs 16-byte aligned source and size\n"); std::abort(); }
  std::lock_guard<std::mutex> lk(emu::copy_mu);
  const uintptr_t d0 = (uintptr_t)smem_dst, d1 = d0 + bytes;
  for (auto& c : emu::copies) {
    const uintptr_t c0 = (uintptr_t)c.second.dst, c1 = c0 + c.second.bytes;
    if (d0 < c1 && c0 < d1) { std::fprintf(stderr, "emu: cp.async.bulk into a buffer whose previous copy is still outstanding\n"); std::abort(); }
  }
  std::memset(smem_dst, 0xFF, bytes);
  emu::copies.push_back({bar, emu::PendingCopy{smem_dst, gmem_src, bytes, emu::copy_delay(bar)}});
}
