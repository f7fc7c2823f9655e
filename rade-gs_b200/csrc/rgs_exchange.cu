// rgs_exchange.cu -- multi-GPU exchange of the screen-space gradient rows over peer memory (NVLink / NVSwitch).
//
// One process per GPU; every rank renders a slab of tile rows, so its accumulator rows are non-zero only for the splats
// that reach its slab.  The exchange that the north star places after backward-render ("one all-reduce of the
// per-Gaussian gradients") is done here on the device instead of by a host-driven dense NCCL all-reduce:
//
//   every rank owns a contiguous block of Gaussian rows (owner = idx / rows_per_rank) and exposes ONE device allocation
//   (cudaMalloc + cudaIpcGetMemHandle; peers map it with cudaIpcOpenMemHandle) holding
//       sum  [rows_per_rank][row]   reduce target of the rows it owns
//       full [capacity][row]        the summed rows of ALL Gaussians, as backward-preprocess reads them
//       flags[world]                barrier epochs written by the peers
//       mark [rows_per_rank]        one byte per owned row: somebody pushed into it this step
//   1. push   : a rank walks the rows its slab touched (tiles_touched > 0), adds each non-zero row into the OWNER's `sum`
//               with 16-byte vector reductions straight through NVLink (red.global.add.v4.f32 on the peer mapping), and
//               clears its local row (the local accumulator is persistent: no 64..384 MB memset per step);
//   2. barrier: release/acquire flags in peer memory, one tiny kernel, no host involvement;
//   3. spread : the owner writes every summed row whose content changed to the `full` array of every rank (plain 16-byte
//               stores over NVLink) and clears its `sum` row for the next step;
//   4. barrier, then backward-preprocess reads the local `full`.
// Every rank ends with bit-identical rows (one sum per row, computed at its owner, copied everywhere): replicated
// optimiser states cannot drift apart, which a "everybody adds into everybody" scheme would not guarantee.
// Traffic per rank and step: pushed rows (~1.25/world of the visible splats at 8 ranks) + its share of the summed rows to
// world-1 peers, instead of 2 x (world-1)/world of the dense P x row tensor through NCCL's ring -- and no host
// synchronisation, size exchange or staging copy.  Reference: none (the reference is single-GPU); the semantics matched
// are those of the atomic accumulation in backward.cu:878-1013 (a sum over pixels, here over slabs as well).
#include <cstdio>
#include <cstring>
#include <string>

#include "rgs_common.cuh"

namespace rgs {

constexpr int MAX_WORLD = 16;

struct PeerTable {
	float* sum[MAX_WORLD];
	float* full[MAX_WORLD];
	uint32_t* flags[MAX_WORLD];
	uint8_t* mark[MAX_WORLD];  // [rows_per_rank_cap] per owned row: some rank pushed into it this step
};

}  // namespace rgs

struct rgs_exchange {
	int rank, world, device;
	int64_t capacity;
	int row_floats;
	int64_t rows_per_rank_cap;
	char* base;                 // own window
	size_t bytes, off_full, off_flags, off_mark;
	char* peer_base[rgs::MAX_WORLD];
	bool connected;
	rgs::PeerTable tab;
	float* acc_local;           // persistent local accumulator [capacity][row], kept all-zero between steps
	uint8_t* dirty;             // [rows_per_rank_cap] owner-side: row was non-zero in `full` after the previous step
	uint32_t epoch;
	int64_t last_P;
};

namespace rgs {

// One thread per Gaussian finds the rows this rank's slab touched (coalesced read of the per-splat tile counts); the rows found by a
// warp are then handled one after the other by its first RQ lanes (RQ = float4 per row, 4 or 8): read the local row, clear it
// (self-cleaning accumulator), add the non-zero quarters into the OWNER's `sum` row over NVLink and raise the owner's per-row mark so
// that its spread pass looks at this row.  (A thread per 16 bytes, as first written, made the kernel thread-count bound: 0.4-0.5 ms at
// 3-10 M Gaussians although only a few per cent of the rows carry anything.)
template <int RQ>
__global__ void __launch_bounds__(256) exchange_push_kernel(int P, int rows_per_rank, float4* __restrict__ acc_local,
                                                            const uint32_t* __restrict__ tiles_touched, PeerTable tab) {
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	const int lane = threadIdx.x & 31;
	const bool touched = idx < P && tiles_touched[idx] != 0;
	unsigned m = __ballot_sync(0xffffffffu, touched);
	while (m) {
		const int rid = idx - lane + (__ffs(m) - 1);
		m &= m - 1;
		bool nz = false;
		if (lane < RQ) {
			float4* src = acc_local + (size_t)rid * RQ + lane;
			const float4 v = *src;
			nz = !(v.x == 0.f && v.y == 0.f && v.z == 0.f && v.w == 0.f);
			if (nz) {
				*src = make_float4(0.f, 0.f, 0.f, 0.f);
				const int owner = rid / rows_per_rank;
				red_add_v4(tab.sum[owner] + ((size_t)(rid - owner * rows_per_rank) * RQ + lane) * 4, v);
			}
		}
		const unsigned any_nz = __ballot_sync(0xffffffffu, nz);
		if (any_nz != 0 && lane == 0) {
			const int owner = rid / rows_per_rank;
			tab.mark[owner][rid - owner * rows_per_rank] = 1;   // idempotent byte store into the owner's window
		}
	}
}

// All-to-all barrier through flags in peer memory: thread p tells peer p "rank `rank` reached `epoch`", then waits until
// peer p said the same here.  Everything this rank wrote before (previous kernels on the stream) is ordered before the flag
// by the system-scope fence + release store; the acquire load orders the peers' data before whatever follows.
__global__ void exchange_barrier_kernel(int rank, int world, uint32_t epoch, PeerTable tab, int* __restrict__ timeout_flag) {
	const int p = threadIdx.x;
	__threadfence_system();
	if (p < world) {
		uint32_t* remote = tab.flags[p] + rank;
		asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(remote), "r"(epoch) : "memory");
		const uint32_t* mine = tab.flags[rank] + p;
		const long long t0 = clock64();
		uint32_t seen;
		do {
			asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(mine) : "memory");
			if ((int32_t)(seen - epoch) >= 0) break;
			if (clock64() - t0 > 20000000000ll) {  // ~10 s at 2 GHz: a peer never arrived.  Do not hang the box and do not kill the
				*timeout_flag = 1 + p;             // context either: raise the flag (rgs_exchange_status reports it) and carry on --
				__threadfence_system();            // the rows of this step are then meaningless, which the caller must check for
				break;
			}
			__nanosleep(200);
		} while (true);
	}
	__threadfence_system();
}

// The owner's pass: one thread per owned row reads its mark (set by the pushers) and its dirty flag (row was non-zero in `full`
// after the previous step); the rows found by a warp are copied, RQ lanes at a time, from `sum` to the `full` array of EVERY rank
// (world plain stores) and `sum` is cleared.  Rows that carried something last step and nothing now are
// rewritten with zeros once.
template <int RQ>
__global__ void __launch_bounds__(256) exchange_spread_kernel(int P, int rows_per_rank, int rank, int world, float4* __restrict__ my_sum,
                                                              uint8_t* __restrict__ dirty, uint8_t* __restrict__ my_mark, PeerTable tab) {
	const int local = blockIdx.x * blockDim.x + threadIdx.x;
	const int lane = threadIdx.x & 31;
	const bool valid = local < rows_per_rank && rank * rows_per_rank + local < P;
	const bool work = valid && ((my_mark[local] | dirty[local]) != 0);
	unsigned m = __ballot_sync(0xffffffffu, work);
	while (m) {
		const int l = local - lane + (__ffs(m) - 1);
		m &= m - 1;
		const size_t idx = (size_t)rank * rows_per_rank + l;
		bool nz = false;
		if (lane < RQ) {
			float4* src = my_sum + (size_t)l * RQ + lane;
			const float4 v = *src;
			// on the bits, not `== 0`: red.add.f32 flushes a subnormal sum to -0.0, which must be cleared from `sum` and
			// rewritten as +0.0 in `full` next step like any other value
			nz = (__float_as_uint(v.x) | __float_as_uint(v.y) | __float_as_uint(v.z) | __float_as_uint(v.w)) != 0u;
			if (nz) *src = make_float4(0.f, 0.f, 0.f, 0.f);
			for (int p = 0; p < world; p++) reinterpret_cast<float4*>(tab.full[p])[idx * RQ + lane] = v;
		}
		const unsigned row_nz = __ballot_sync(0xffffffffu, nz);
		if (lane == 0) {
			dirty[l] = row_nz != 0 ? 1 : 0;
			my_mark[l] = 0;
		}
	}
}

}  // namespace rgs

using namespace rgs;

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static void layout(rgs_exchange* ex) {
	const size_t row = (size_t)ex->row_floats * sizeof(float);
	ex->rows_per_rank_cap = (ex->capacity + ex->world - 1) / ex->world;
	ex->off_full = align_up((size_t)ex->rows_per_rank_cap * row, 256);
	ex->off_flags = ex->off_full + align_up((size_t)ex->capacity * row, 256);
	ex->off_mark = ex->off_flags + 256;
	ex->bytes = ex->off_mark + align_up((size_t)ex->rows_per_rank_cap, 256);
}

// The window, the local accumulator and the dirty flags, zeroed, and the window's IPC handle into `ipc_handle`.
static int allocate(rgs_exchange* ex, void* ipc_handle) {
	RGS_CUDA_TRY(cudaGetDevice(&ex->device));
	layout(ex);
	const size_t row = (size_t)ex->row_floats * sizeof(float);
	RGS_CUDA_TRY(cudaMalloc((void**)&ex->base, ex->bytes));
	RGS_CUDA_TRY(cudaMemset(ex->base, 0, ex->bytes));
	RGS_CUDA_TRY(cudaMalloc((void**)&ex->acc_local, (size_t)ex->capacity * row));
	RGS_CUDA_TRY(cudaMemset(ex->acc_local, 0, (size_t)ex->capacity * row));
	RGS_CUDA_TRY(cudaMalloc((void**)&ex->dirty, (size_t)ex->rows_per_rank_cap));
	RGS_CUDA_TRY(cudaMemset(ex->dirty, 0, (size_t)ex->rows_per_rank_cap));
	RGS_CUDA_TRY(cudaDeviceSynchronize());
	cudaIpcMemHandle_t h;
	static_assert(sizeof(h) == RGS_IPC_HANDLE_BYTES, "IPC handle size");
	RGS_CUDA_TRY(cudaIpcGetMemHandle(&h, ex->base));
	memcpy(ipc_handle, &h, sizeof(h));
	return RGS_OK;
}

extern "C" {

int32_t rgs_exchange_create(int32_t rank, int32_t world, int64_t capacity_rows, int32_t row_floats, rgs_exchange** out, void* ipc_handle) {
	if (!out || !ipc_handle) return fail(RGS_E_INVALID, "null pointer");
	if (world < 1 || world > MAX_WORLD || rank < 0 || rank >= world) return fail(RGS_E_INVALID, "rank / world out of range (world <= 16)");
	if (capacity_rows <= 0 || (row_floats != GRAD_FLOATS_BASE && row_floats != GRAD_FLOATS_COORD)) return fail(RGS_E_INVALID, "capacity / row size");
	rgs_exchange* ex = new rgs_exchange();
	memset(ex, 0, sizeof(*ex));
	ex->rank = rank; ex->world = world; ex->capacity = capacity_rows; ex->row_floats = row_floats;
	ex->last_P = -1;
	const int rc = allocate(ex, ipc_handle);
	if (rc != RGS_OK) {
		rgs_exchange_destroy(ex);   // frees what was allocated before the failing call
		return rc;
	}
	*out = ex;
	return RGS_OK;
}

int32_t rgs_exchange_connect(rgs_exchange* ex, const void* all_handles) {
	if (!ex || !all_handles) return fail(RGS_E_INVALID, "null pointer");
	if (ex->connected) return fail(RGS_E_INVALID, "already connected");
	for (int p = 0; p < ex->world; p++) {
		if (p == ex->rank) {
			ex->peer_base[p] = ex->base;
		} else {
			cudaIpcMemHandle_t h;
			memcpy(&h, (const char*)all_handles + (size_t)p * RGS_IPC_HANDLE_BYTES, sizeof(h));
			void* ptr = nullptr;
			RGS_CUDA_TRY(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
			ex->peer_base[p] = (char*)ptr;
		}
		ex->tab.sum[p] = reinterpret_cast<float*>(ex->peer_base[p]);
		ex->tab.full[p] = reinterpret_cast<float*>(ex->peer_base[p] + ex->off_full);
		ex->tab.flags[p] = reinterpret_cast<uint32_t*>(ex->peer_base[p] + ex->off_flags);
		ex->tab.mark[p] = reinterpret_cast<uint8_t*>(ex->peer_base[p] + ex->off_mark);
	}
	ex->connected = true;
	return RGS_OK;
}

int32_t rgs_exchange_destroy(rgs_exchange* ex) {
	if (!ex) return RGS_OK;
	cudaDeviceSynchronize();
	for (int p = 0; p < ex->world; p++)   // also the windows a failed rgs_exchange_connect opened before its failure
		if (p != ex->rank && ex->peer_base[p]) cudaIpcCloseMemHandle(ex->peer_base[p]);
	cudaFree(ex->base);
	cudaFree(ex->acc_local);
	cudaFree(ex->dirty);
	delete ex;
	return RGS_OK;
}

float* rgs_exchange_accumulator(rgs_exchange* ex) { return ex ? ex->acc_local : nullptr; }
const float* rgs_exchange_result(rgs_exchange* ex) { return ex ? reinterpret_cast<const float*>(ex->base + ex->off_full) : nullptr; }

// pinned flag the barrier kernel raises before trapping, so the host can say WHICH peer never arrived
static int* timeout_flag() {
	static thread_local int* f = nullptr;
	if (!f) {
		if (cudaHostAlloc((void**)&f, 64, cudaHostAllocMapped) != cudaSuccess) return nullptr;
		*f = 0;
	}
	return f;
}

int32_t rgs_exchange_rows(rgs_exchange* ex, int32_t P, const uint32_t* tiles_touched, const int32_t* radii, void* cuda_stream) {
	if (!ex || !ex->connected) return fail(RGS_E_INVALID, "exchange not connected");
	if (P < 0 || P > ex->capacity) return fail(RGS_E_INVALID, "more Gaussians than the exchange was created for: re-create it (collectively) with a larger capacity");
	if (P == 0) return RGS_OK;
	if (!tiles_touched || !radii) return fail(RGS_E_INVALID, "null pointer");
	cudaStream_t s = (cudaStream_t)cuda_stream;
	int* tf = timeout_flag();
	if (!tf) return fail(RGS_E_CUDA, "cudaHostAlloc failed");
	if (*tf) return fail(RGS_E_CUDA, "a previous exchange barrier timed out waiting for rank " + std::to_string(*tf - 1));
	const int rq = ex->row_floats / 4;
	const int rows_per_rank = (P + ex->world - 1) / ex->world;
	if (P != ex->last_P) {
		// the row <-> Gaussian association changed (densification, first call): forget what `full` held.  Every rank sees the
		// same sequence of P, so all do this in the same step; peers write into `full` only after the next barrier.
		RGS_CUDA_TRY(cudaMemsetAsync(ex->base + ex->off_full, 0, (size_t)ex->capacity * ex->row_floats * sizeof(float), s));
		RGS_CUDA_TRY(cudaMemsetAsync(ex->dirty, 0, (size_t)ex->rows_per_rank_cap, s));
		ex->last_P = P;   // (marks and `sum` are always left clear by the spread pass)
	}
	{
		const unsigned blocks = (unsigned)((P + 255) / 256);
		if (rq == 4) exchange_push_kernel<4><<<blocks, 256, 0, s>>>(P, rows_per_rank, reinterpret_cast<float4*>(ex->acc_local), tiles_touched, ex->tab);
		else exchange_push_kernel<8><<<blocks, 256, 0, s>>>(P, rows_per_rank, reinterpret_cast<float4*>(ex->acc_local), tiles_touched, ex->tab);
	}
	exchange_barrier_kernel<<<1, 32, 0, s>>>(ex->rank, ex->world, ++ex->epoch, ex->tab, tf);
	{
		const unsigned blocks = (unsigned)((rows_per_rank + 255) / 256);
		float4* my_sum = reinterpret_cast<float4*>(ex->base);
		uint8_t* my_mark = reinterpret_cast<uint8_t*>(ex->base + ex->off_mark);
		if (rq == 4) exchange_spread_kernel<4><<<blocks, 256, 0, s>>>(P, rows_per_rank, ex->rank, ex->world, my_sum, ex->dirty, my_mark, ex->tab);
		else exchange_spread_kernel<8><<<blocks, 256, 0, s>>>(P, rows_per_rank, ex->rank, ex->world, my_sum, ex->dirty, my_mark, ex->tab);
	}
	exchange_barrier_kernel<<<1, 32, 0, s>>>(ex->rank, ex->world, ++ex->epoch, ex->tab, tf);
	count_launch(4);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) return fail(RGS_E_CUDA, cudaGetErrorString(e));
	return RGS_OK;
}

// 0 = healthy; 1 + p = a barrier gave up waiting for rank p (after synchronising the stream the exchange ran on).
int32_t rgs_exchange_status(rgs_exchange* ex, void* cuda_stream) {
	if (!ex) return fail(RGS_E_INVALID, "null exchange");
	cudaError_t e = cudaStreamSynchronize((cudaStream_t)cuda_stream);
	if (e != cudaSuccess) return fail(RGS_E_CUDA, cudaGetErrorString(e));
	int* tf = timeout_flag();
	return tf ? *tf : 0;
}

}  // extern "C"
