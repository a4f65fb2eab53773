// ipc_probe.cu -- feasibility + latency probe for the peer-memory data plane of the multi-GPU engine (tools only).
// Forks one process per GPU (like torchrun does), exchanges cudaIpcMemHandles over pipes, maps every peer's window and
// measures (a) a flag ping-pong between GPU 0 and GPU 1 driven entirely from kernels (store to peer + spin on local),
// (b) the bandwidth of a kernel that copies a buffer into peer memory with plain coalesced stores.
//   nvcc -O2 -gencode arch=compute_90a,code=sm_90a -o tools/ipc_probe tools/ipc_probe.cu && tools/ipc_probe 2
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <unistd.h>
#include <sys/wait.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { fprintf(stderr, "[rank %d] %s: %s\n", g_rank, #x, cudaGetErrorString(e)); exit(2); } } while (0)
static int g_rank = -1;

__global__ void k_pingpong(volatile unsigned long long* mine, volatile unsigned long long* peer, int rank, int iters) {
    // rank 0 sends i, waits for i back; rank 1 waits for i, sends i back
    for (int i = 1; i <= iters; i++) {
        if (rank == 0) {
            *peer = (unsigned long long) i;
            __threadfence_system();
            while (*mine < (unsigned long long) i) { }
        }
        else {
            while (*mine < (unsigned long long) i) { }
            *peer = (unsigned long long) i;
            __threadfence_system();
        }
    }
}

__global__ void k_copy(const uint4* src, uint4* dst, size_t n) {
    for (size_t i = blockIdx.x*(size_t) blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x*blockDim.x) dst[i] = src[i];
}

// many small CTAs, each stores `per` float4 to the target (coalesced or strided by 3), then fences at system scope
// (every thread, or thread 0 after a barrier) and bumps a local counter: the pattern of k_integrate / k_force_push
__global__ void k_small_stores(float4* dst, int per, int strided, int fenceAll, unsigned int* done) {
    const int base = blockIdx.x*per*(strided ? 3 : 1);
    for (int i = threadIdx.x; i < per; i += blockDim.x) dst[base + (strided ? 3*i : i)] = make_float4(i, 1.f, 2.f, 3.f);
    if (fenceAll) __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) { if (!fenceAll) __threadfence_system(); atomicAdd(done, 1u); }
}

static void xwrite(int fd, const void* p, size_t n) { if (write(fd, p, n) != (ssize_t) n) { perror("write"); exit(3); } }
static void xread(int fd, void* p, size_t n) { size_t got = 0; while (got < n) { ssize_t r = read(fd, (char*) p + got, n - got); if (r <= 0) { perror("read"); exit(3); } got += r; } }

int main(int argc, char** argv) {
    const int world = argc > 1 ? atoi(argv[1]) : 2;
    // pipes[a][b]: a writes, b reads
    std::vector<std::vector<int> > rd(world, std::vector<int>(world)), wr(world, std::vector<int>(world));
    for (int a = 0; a < world; a++) for (int b = 0; b < world; b++) { int fd[2]; if (pipe(fd)) return 1; rd[a][b] = fd[0]; wr[a][b] = fd[1]; }
    std::vector<pid_t> kids;
    for (int r = 0; r < world; r++) {
        pid_t pid = fork();
        if (pid == 0) { g_rank = r; break; }
        kids.push_back(pid);
    }
    if (g_rank < 0) {
        int bad = 0;
        for (pid_t k : kids) { int st; waitpid(k, &st, 0); if (!WIFEXITED(st) || WEXITSTATUS(st)) bad = 1; }
        printf("ipc_probe: %s\n", bad ? "FAILED" : "ok");
        return bad;
    }
    const int rank = g_rank;
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));
    if (ndev < world) { fprintf(stderr, "need %d devices, have %d\n", world, ndev); return 2; }
    CK(cudaSetDevice(rank));
    const size_t bytes = 64u << 20;
    char* win = nullptr;
    CK(cudaMalloc(&win, bytes));
    CK(cudaMemset(win, 0, bytes));
    cudaIpcMemHandle_t mine;
    CK(cudaIpcGetMemHandle(&mine, win));
    for (int q = 0; q < world; q++) if (q != rank) xwrite(wr[rank][q], &mine, sizeof(mine));
    std::vector<char*> peer(world, nullptr);
    for (int q = 0; q < world; q++) {
        if (q == rank) { peer[q] = win; continue; }
        cudaIpcMemHandle_t h;
        xread(rd[q][rank], &h, sizeof(h));
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, rank, q));
        CK(cudaIpcOpenMemHandle((void**) &peer[q], h, cudaIpcMemLazyEnablePeerAccess));
        if (rank == 0) printf("rank 0: canAccessPeer(%d) = %d, mapped %p\n", q, can, (void*) peer[q]);
    }
    // barrier over pipes
    auto barrier = [&]() { char c = 1; for (int q = 0; q < world; q++) if (q != rank) xwrite(wr[rank][q], &c, 1); for (int q = 0; q < world; q++) if (q != rank) xread(rd[q][rank], &c, 1); };
    barrier();
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    if (rank < 2) {
        const int iters = 20000;
        const int other = 1 - rank;
        CK(cudaEventRecord(e0));
        k_pingpong<<<1, 1>>>((volatile unsigned long long*) win, (volatile unsigned long long*) peer[other], rank, iters);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (rank == 0) printf("flag ping-pong GPU0<->GPU1: %.2f us per round trip (%.2f us one way)\n", 1e3*ms/iters, 0.5e3*ms/iters);
    }
    barrier();
    // bandwidth: every rank writes 32 MiB into its right neighbour's window at offset 16 MiB
    {
        const size_t n = (32u << 20)/16;
        char* src = nullptr;
        CK(cudaMalloc(&src, 32u << 20));
        CK(cudaMemset(src, rank + 1, 32u << 20));
        const int to = (rank + 1) % world;
        for (int rep = 0; rep < 3; rep++) k_copy<<<132*4, 256>>>((const uint4*) src, (uint4*) (peer[to] + (16u << 20)), n);
        CK(cudaDeviceSynchronize());
        barrier();
        CK(cudaEventRecord(e0));
        for (int rep = 0; rep < 10; rep++) k_copy<<<132*4, 256>>>((const uint4*) src, (uint4*) (peer[to] + (16u << 20)), n);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
        printf("rank %d -> %d: store bandwidth %.1f GB/s (32 MiB x 10, all ranks at once)\n", rank, to, 10.0*(32u << 20)/(ms*1e-3)/1e9);
        // small transfers: 256 KiB
        const size_t ns = (256u << 10)/16;
        CK(cudaEventRecord(e0));
        for (int rep = 0; rep < 100; rep++) k_copy<<<64, 256>>>((const uint4*) src, (uint4*) (peer[to] + (16u << 20)), ns);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if (rank == 0) printf("rank 0: 256 KiB store kernel %.2f us each (back to back)\n", 1e3*ms/100);
        barrier();
        // verify what the left neighbour wrote
        unsigned char probe = 0;
        CK(cudaMemcpy(&probe, win + (16u << 20) + 12345, 1, cudaMemcpyDeviceToHost));
        const int from = (rank + world - 1) % world;
        if (probe != (unsigned char) (from + 1)) { fprintf(stderr, "rank %d: wrong data from %d: %d\n", rank, from, probe); return 4; }
    }
    barrier();
    // small-store kernels: 180 CTAs x 64 threads x 192 float4 (3 KB per CTA), local vs peer target
    {
        unsigned int* done = nullptr;
        CK(cudaMalloc(&done, 4)); CK(cudaMemset(done, 0, 4));
        const int to = (rank + 1) % world;
        for (int target = 0; target < 2; target++) for (int strided = 0; strided < 2; strided++) for (int fenceAll = 0; fenceAll < 2; fenceAll++) {
            float4* dst = (float4*) ((target ? peer[to] : win) + (16u << 20));
            for (int rep = 0; rep < 3; rep++) k_small_stores<<<180, 64>>>(dst, 192, strided, fenceAll, done);
            CK(cudaDeviceSynchronize());
            barrier();
            CK(cudaEventRecord(e0));
            for (int rep = 0; rep < 20; rep++) k_small_stores<<<180, 64>>>(dst, 192, strided, fenceAll, done);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
            if (rank == 0) printf("small stores: %s target, %s, fence by %s: %.2f us per kernel\n", target ? "PEER" : "local", strided ? "stride 3" : "coalesced", fenceAll ? "every thread" : "thread 0", 1e3*ms/20);
            barrier();
        }
    }
    barrier();
    for (int q = 0; q < world; q++) if (q != rank) cudaIpcCloseMemHandle(peer[q]);
    return 0;
}
