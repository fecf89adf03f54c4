// ptx.cuh -- thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, wgmma (warpgroup MMA, shared-memory descriptors), async-proxy fences, TMA, f16x2 / f32 reductions.
// Everything here is sm_90a-only by design (no fallback paths).
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace tcnnb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
	return (uint32_t)__cvta_generic_to_shared(p);
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}

__device__ __forceinline__ void fence_mbar_init() {
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"WAIT_LOOP:\n"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
		"@p bra WAIT_DONE;\n"
		"bra WAIT_LOOP;\n"
		"WAIT_DONE:\n"
		"}\n" ::"r"(bar), "r"(parity)
		: "memory");
}

// ---------------------------------------------------------------- proxies / fences
// Make generic-proxy shared-memory writes visible to the async proxy (wgmma operand reads).
__device__ __forceinline__ void fence_proxy_async_smem() {
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor, SWIZZLE_128B canonical layouts (tile rows are 128 bytes = 64 fp16):
//   bits [ 0,14) start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type: 1 = SWIZZLE_128B
// K-major operand  ([rows = M/N][64 K-elements]):  SBO = 1024 B (next group of 8 rows), LBO unused (1); the k-th step of 16 elements
//   starts 32 k bytes into the row (the hardware applies the swizzle to the computed addresses).
// MN-major operand ([rows = K][64 MN-elements]):   SBO = 1024 B (next group of 8 K-rows), LBO = stride between
//   64-element blocks along MN (only read when the MN extent exceeds 64).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
	uint64_t d = 0;
	d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
	d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
	d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
	d |= (uint64_t)1 << 62;
	return d;
}

// Orders the warpgroup's register / shared-memory accesses before the wgmma instructions that follow.
__device__ __forceinline__ void wgmma_fence() {
	asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}

__device__ __forceinline__ void wgmma_commit() {
	asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}

// Wait until at most N committed groups of this warp are pending.
template <int N>
__device__ __forceinline__ void wgmma_wait() {
	asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// Pins the accumulator registers at this point of the program: the compiler must not move their reads above a wgmma_wait.
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
	for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] . B[16 x N], fp16 operands, fp32 accumulators in registers (scale_d = 0: D is overwritten).
//   ss: A and B from shared memory (descriptors); TA / TB = 1: the operand is MN-major (transposed).
//   rs: A from registers in the accumulator-compatible fragment layout (thread (warp w, lane l) holds rows 16 w + l / 4 and + 8,
//       columns 2 (l % 4) + {0, 1} and + 8, as packed fp16 pairs a[0..3] = (r, c), (r + 8, c), (r, c + 8), (r + 8, c + 8)).
// Accumulator fragment: d[4 i + {0, 1}] = row 16 w + l / 4, columns 8 i + 2 (l % 4) + {0, 1}; d[4 i + {2, 3}] = the row 8 below.
template <int N>
struct Wgmma;

template <>
struct Wgmma<16> {
	template <int TA, int TB>
	__device__ __forceinline__ static void ss(float (&d)[8], uint64_t a, uint64_t b, uint32_t scale_d) {
		asm volatile(
			"{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
			"wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
			: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
			: "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
	}
	template <int TB>
	__device__ __forceinline__ static void rs(float (&d)[8], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
		asm volatile(
			"{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
			"wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, %14;\n}\n"
			: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
			: "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB));
	}
};

template <>
struct Wgmma<32> {
	template <int TA, int TB>
	__device__ __forceinline__ static void ss(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
		asm volatile(
			"{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
			"wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
			: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
			: "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
	}
	template <int TB>
	__device__ __forceinline__ static void rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
		asm volatile(
			"{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
			"wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, %22;\n}\n"
			: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
			: "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB));
	}
};

template <>
struct Wgmma<64> {
	template <int TA, int TB>
	__device__ __forceinline__ static void ss(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
		asm volatile(
			"{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
			"wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
			: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
			: "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
	}
	template <int TB>
	__device__ __forceinline__ static void rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
		asm volatile(
			"{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
			"wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n}\n"
			: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
			: "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB));
	}
};

template <>
struct Wgmma<128> {
	template <int TA, int TB>
	__device__ __forceinline__ static void ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
		asm volatile(
			"{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
			"wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
			: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
			: "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
	}
	template <int TB>
	__device__ __forceinline__ static void rs(float (&d)[64], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
		asm volatile(
			"{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
			"wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, %70;\n}\n"
			: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
			: "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB));
	}
};

// ---------------------------------------------------------------- mbarrier extras + TMA (cp.async.bulk.tensor)
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
	uint32_t ok;
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
		"selp.u32 %0, 1, 0, p;\n"
		"}\n"
		: "=r"(ok)
		: "r"(bar), "r"(parity)
		: "memory");
	return ok != 0;
}

__device__ __forceinline__ void mbar_arrive_plain(uint32_t bar) {
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

// 2-D tiled TMA load global -> shared (tensor map in kernel parameter / constant space), completion on an mbarrier.
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tensor_map, uint32_t bar, int32_t x, int32_t y) {
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_dst), "l"(tensor_map), "r"(bar), "r"(x),
	             "r"(y)
	             : "memory");
}

__device__ __forceinline__ void tma_prefetch_desc(const void* tensor_map) {
	asm volatile("prefetch.tensormap [%0];" ::"l"(tensor_map) : "memory");
}

// ---------------------------------------------------------------- global reductions
// red.global.add.noftz.f16x2: the same instruction the reference's atomic_add_gmem(__half2) lowers to (vec.h:328-336).
__device__ __forceinline__ void red_add_f16x2(__half2* addr, __half2 v) {
	asm volatile("red.relaxed.gpu.global.add.noftz.f16x2 [%0], %1;" ::"l"(addr), "r"(*reinterpret_cast<uint32_t*>(&v)) : "memory");
}

__device__ __forceinline__ void red_add_f32(float* addr, float v) {
	asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}

// 8- / 16-byte vector reductions (sm_90+): two / four fp32 adds in one L2 operation; the address must be 8- / 16-byte aligned.
__device__ __forceinline__ void red_add_v2_f32(float* addr, float a, float b) {
	asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

__device__ __forceinline__ void red_add_v4_f32(float* addr, float a, float b, float c, float d) {
	asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

}  // namespace ptx
}  // namespace tcnnb
