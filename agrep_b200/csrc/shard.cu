/* agrep_b200/csrc/shard.cu -- one text over several GPUs (SURVEY 8e): the C side of the sharded scan.
 *
 * One process per GPU; every rank holds a byte range of the text in its HBM.  Records are independent once their
 * boundaries are known (the automaton is reset at every delimiter, asearch.c:175-196), so the scan itself needs no
 * collective.  What the ranks exchange:
 *   - once per text, 64.5 KiB of halo with each neighbour (agb_shard_halo: ncclSend/ncclRecv), so that the cut rule can
 *     run on the device: a shard's scan starts AGB_HALO_LEFT bytes early -- a delimiter that straddles the cut, or a run
 *     of "$$", is parsed as it is in the whole text -- and runs into the next shard until the record in progress closes;
 *     a record belongs to the shard that holds the last byte of the delimiter that opened it (RecParams.own_lo/own_hi,
 *     applied where the record stage decides what counts);
 *   - per scan, a 256-byte header per rank (ncclAllGather: counts, level histogram, delimiter counts for the ordinals,
 *     list length) and the match lists padded to the longest (one more ncclAllGather); a kernel then writes the ordered
 *     list of the whole text with global offsets and ordinals.  Two host synchronisations per scan: the local result and
 *     the gathered headers.
 */
#include "scan_internal.cuh"
#include "automaton.cuh"
#include <nccl.h>
#include <dlfcn.h>

/* NCCL is bound at run time, not at link time: a process that also runs PyTorch must end up with ONE libnccl.so.2, and
 * PyTorch brings its own (newer) one -- had this library the system's as a link-time dependency, importing it first would
 * pin that older one under the same soname and libtorch_cuda.so would fail to resolve its symbols.  dlopen() by soname
 * returns whatever copy is already loaded, else the system's. */
static struct NcclApi {
	void *h;
	ncclResult_t (*GetUniqueId)(ncclUniqueId *);
	ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int);
	ncclResult_t (*CommDestroy)(ncclComm_t);
	ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
	ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
	ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
	ncclResult_t (*GroupStart)(void);
	ncclResult_t (*GroupEnd)(void);
	const char *(*GetErrorString)(ncclResult_t);
} g_nccl;

static int nccl_load(void)
{
	if (g_nccl.h) return AGB_OK;
	void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
	if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
	if (!h) { snprintf(g_err, sizeof g_err, "NCCL is not available: %s", dlerror()); return AGB_ERR_CUDA; }
#define NCCL_SYM(field, name) do { *(void **)(&g_nccl.field) = dlsym(h, name); if (!g_nccl.field) { snprintf(g_err, sizeof g_err, "libnccl lacks %s", name); return AGB_ERR_CUDA; } } while (0)
	NCCL_SYM(GetUniqueId, "ncclGetUniqueId"); NCCL_SYM(CommInitRank, "ncclCommInitRank"); NCCL_SYM(CommDestroy, "ncclCommDestroy");
	NCCL_SYM(AllGather, "ncclAllGather"); NCCL_SYM(Send, "ncclSend"); NCCL_SYM(Recv, "ncclRecv");
	NCCL_SYM(GroupStart, "ncclGroupStart"); NCCL_SYM(GroupEnd, "ncclGroupEnd"); NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef NCCL_SYM
	g_nccl.h = h;
	return AGB_OK;
}
#define ncclGetUniqueId    g_nccl.GetUniqueId
#define ncclCommInitRank   g_nccl.CommInitRank
#define ncclCommDestroy    g_nccl.CommDestroy
#define ncclAllGather      g_nccl.AllGather
#define ncclSend           g_nccl.Send
#define ncclRecv           g_nccl.Recv
#define ncclGroupStart     g_nccl.GroupStart
#define ncclGroupEnd       g_nccl.GroupEnd
#define ncclGetErrorString g_nccl.GetErrorString

#define NCCL_TRY(x) do { ncclResult_t r_ = (x); if (r_ != ncclSuccess) { \
	snprintf(g_err, sizeof g_err, "%s failed: %s (%s:%d)", #x, ncclGetErrorString(r_), __FILE__, __LINE__); \
	return AGB_ERR_CUDA; } } while (0)

#define SHARD_MAXWORLD 64
#define HDR_WORDS 32            /* u64 per rank */
enum { H_MATCHED = 0, H_RECORDS = 1, H_FLAGGED = 2, H_HIST = 3 /* ..11 */, H_CLOSES = 12 /* delimiter ends inside the shard's own range */,
       H_ORD_FIX = 13 /* what the shard's local ordinals count that is not its own */, H_ORD_ORIGIN = 14 /* rank 0: j before the first byte */,
       H_TRUNC = 15, H_NLOCAL = 16, H_MS_FRONT = 17, H_MS_REC = 18, H_VIRT = 19 /* rank 0: 1 when the virtual '\n' closes a record of its own */ };

struct agb_comm {
	ncclComm_t nccl; int world, rank, dev;
	uint64_t sizes[SHARD_MAXWORLD];           /* n_local of every rank (agb_shard_halo) */
	uint64_t halo_left, halo_right; int reaches_end; bool halo_known;
	unsigned long long *d_hdr, *d_all;        /* device: own header, all headers */
	unsigned long long *h_hdr, *h_all;        /* pinned */
	agb_record *d_local, *d_pad; uint64_t local_cap, pad_cap;
};

extern "C" int agb_comm_unique_id(void *id128)
{
	ncclUniqueId id;
	if (!id128) return AGB_ERR_ARG;
	{ int rc = nccl_load(); if (rc) return rc; }
	NCCL_TRY(ncclGetUniqueId(&id));
	static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
	memcpy(id128, &id, sizeof id);
	return AGB_OK;
}

extern "C" int agb_comm_init(agb_comm **out, int world, int rank, const void *id128)
{
	if (!out || !id128 || world < 1 || world > SHARD_MAXWORLD || rank < 0 || rank >= world) return AGB_ERR_ARG;
	{ int rc = nccl_load(); if (rc) return rc; }
	agb_comm *c = new agb_comm; memset(c, 0, sizeof *c);
	c->world = world; c->rank = rank;
	CUDA_TRY(cudaGetDevice(&c->dev));
	ncclUniqueId id; memcpy(&id, id128, sizeof id);
	NCCL_TRY(ncclCommInitRank(&c->nccl, world, id, rank));
	CUDA_TRY(cudaMalloc(&c->d_hdr, HDR_WORDS * sizeof(unsigned long long)));
	CUDA_TRY(cudaMalloc(&c->d_all, (size_t)world * HDR_WORDS * sizeof(unsigned long long)));
	CUDA_TRY(cudaMallocHost(&c->h_hdr, HDR_WORDS * sizeof(unsigned long long)));
	CUDA_TRY(cudaMallocHost(&c->h_all, (size_t)world * HDR_WORDS * sizeof(unsigned long long)));
	*out = c;
	return AGB_OK;
}

extern "C" void agb_comm_free(agb_comm *c)
{
	if (!c) return;
	ncclCommDestroy(c->nccl);
	cudaFree(c->d_hdr); cudaFree(c->d_all); cudaFreeHost(c->h_hdr); cudaFreeHost(c->h_all); cudaFree(c->d_local); cudaFree(c->d_pad);
	delete c;
}
extern "C" int agb_comm_world(const agb_comm *c) { return c ? c->world : 0; }
extern "C" int agb_comm_rank(const agb_comm *c) { return c ? c->rank : -1; }

/* the halos of this rank's shard from its neighbours: the last AGB_HALO_LEFT bytes of the shard before it in front of
 * d_shard, the first AGB_HALO_RIGHT (+16: the scan reads whole 16-byte groups) bytes of the shard behind it after it */
extern "C" int agb_shard_halo(agb_comm *c, void *d_shard, uint64_t n_local, void *stream)
{
	if (!c || (!d_shard && n_local)) return AGB_ERR_ARG;
	cudaStream_t st = (cudaStream_t)stream;
	CUDA_TRY(cudaSetDevice(c->dev));
	c->h_hdr[0] = n_local;
	CUDA_TRY(cudaMemcpyAsync(c->d_hdr, c->h_hdr, sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
	NCCL_TRY(ncclAllGather(c->d_hdr, c->d_all, 1, ncclUint64, c->nccl, st));
	CUDA_TRY(cudaMemcpyAsync(c->h_all, c->d_all, (size_t)c->world * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
	CUDA_TRY(cudaStreamSynchronize(st));
	for (int r = 0; r < c->world; r++) {
		c->sizes[r] = c->h_all[r];
		if (r + 1 < c->world && (c->sizes[r] < AGB_HALO_LEFT || (c->sizes[r] % 512) != 0)) {
			snprintf(g_err, sizeof g_err, "shard %d holds %llu bytes: every shard but the last must be a multiple of 512 bytes", r, (unsigned long long)c->sizes[r]);
			return AGB_ERR_ARG;
		}
	}
	const int r = c->rank;
	uint8_t *sh = (uint8_t *)d_shard;
	const uint64_t next = r + 1 < c->world ? c->sizes[r + 1] : 0;
	c->halo_left = r > 0 ? AGB_HALO_LEFT : 0;
	c->halo_right = std::min<uint64_t>(next, AGB_HALO_RIGHT);
	c->reaches_end = (r + 1 >= c->world) || (r + 2 >= c->world && next <= AGB_HALO_RIGHT);
	const uint64_t give_prev = std::min<uint64_t>(n_local, AGB_HALO_RIGHT);      /* my head, the previous rank's right halo */
	NCCL_TRY(ncclGroupStart());
	if (r > 0) {
		NCCL_TRY(ncclSend(sh, give_prev, ncclUint8, r - 1, c->nccl, st));
		NCCL_TRY(ncclRecv(sh - AGB_HALO_LEFT, AGB_HALO_LEFT, ncclUint8, r - 1, c->nccl, st));
	}
	if (r + 1 < c->world) {
		NCCL_TRY(ncclSend(sh + n_local - AGB_HALO_LEFT, AGB_HALO_LEFT, ncclUint8, r + 1, c->nccl, st));
		NCCL_TRY(ncclRecv(sh + n_local, c->halo_right, ncclUint8, r + 1, c->nccl, st));
	}
	NCCL_TRY(ncclGroupEnd());
	CUDA_TRY(cudaMemsetAsync(sh + n_local + c->halo_right, 0, 16, st));
	CUDA_TRY(cudaStreamSynchronize(st));
	c->halo_known = true;
	return AGB_OK;
}

/* delimiter ends in [0, x) of the local scan, x a multiple of 512, from the block and tile counts the ordinals pass
 * left behind; and the check that a run delimiter ("$$") that reaches the cut begins inside the left halo */
struct RawReader { const uint8_t *t; uint64_t n; __device__ __forceinline__ int get(int64_t p) { return (p < 0 || (uint64_t)p >= n) ? 256 : t[p]; } };

__global__ void k_shard_aux(const uint8_t *text, uint64_t n, const agb_desc *D, const uint16_t *blocks, const uint64_t *tile_off, uint64_t x_lo, uint64_t x_hi, int have_hi,
                            int kind, int delim0, int dfold0, unsigned long long *out /* [0] S(x_lo), [1] S(x_hi), [2] run error */)
{
	if (threadIdx.x || blockIdx.x) return;
	for (int w = 0; w < 2; w++) {
		const uint64_t x = w ? x_hi : x_lo;
		unsigned long long s = 0;
		if (blocks && (w == 0 || have_hi)) {
			const uint64_t blk = x / ORD_BLOCK, tile = x / ORD_TILE;
			s = tile_off[tile];
			for (uint64_t b = tile * (ORD_TILE / ORD_BLOCK); b < blk; b++) s += blocks[b];
		}
		out[w] = s;
	}
	unsigned long long bad = 0;
	if (kind == 1 && x_lo > 0) {
		int64_t p = (int64_t)x_lo - 1;
		while (p >= 0 && (text[p] | dfold0) == delim0) p--;
		if (p < 0) bad = 1;                                 /* the run covers the whole left halo: where it began is unknown */
	}
	if (kind == 2 && x_lo > 0) {
		/* a chain of overlapping occurrences that crosses the cut must begin inside the left halo, clear of its first bytes */
		RawReader R; R.t = text; R.n = n;
		const int L = D->L;
		uint8_t dl[2 * AGB_MAXDELIM + 2], df[2 * AGB_MAXDELIM + 2];
		for (int i = 0; i < L; i++) { df[i] = D->delim_fold[i]; dl[i] = D->delim[i] | df[i]; }
		for (int64_t e = (int64_t)x_lo; e <= (int64_t)x_lo + L - 2; e++)
			if (delim_occurs(R, e, dl, df, L) && delim_chain_first(R, e, dl, df, L) - L + 1 < L) bad = 1;
	}
	out[2] = bad;
}

struct GatherParams {
	int world; uint64_t pad;
	uint64_t count[SHARD_MAXWORLD], out_off[SHARD_MAXWORLD];
	long long byte_base[SHARD_MAXWORLD], ord_add[SHARD_MAXWORLD];
	int ordinals;
};
/* padded per-rank lists -> the ordered list of the whole text: offsets and ordinals made global */
__global__ void __launch_bounds__(256) k_gather_compact(const agb_record *pad, agb_record *out, uint64_t capacity, const GatherParams G)
{
	const int r = blockIdx.y;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < G.count[r]; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t at = G.out_off[r] + i;
		if (at >= capacity) return;
		agb_record rec = pad[(uint64_t)r * G.pad + i];
		rec.begin += G.byte_base[r]; rec.end += G.byte_base[r];
		if (G.ordinals) rec.ordinal += G.ord_add[r];
		out[at] = rec;
	}
}

int shard_aux_enqueue(const agb_desc &d, Workspace &W, const uint8_t *text, uint64_t n, const ShardInfo *sh, bool ordinals, cudaStream_t st)
{
	const bool first = sh->own_lo == INT64_MIN, open_end = sh->own_hi == INT64_MAX;
	k_shard_aux<<<1, 32, 0, st>>>(text, n, W.d_desc, ordinals ? W.ord_blocks : nullptr, W.tile_offsets, first ? 0 : (uint64_t)sh->own_lo,
	                              open_end ? 0 : (uint64_t)sh->own_hi, open_end ? 0 : 1,
	                              d.delim_kind, d.delim[0] | d.delim_fold[0], d.delim_fold[0], W.totals + 16);
	g_launches++;
	CUDA_TRY(cudaGetLastError());
	return AGB_OK;
}

static int comm_buffers(agb_comm *c, uint64_t local_cap, uint64_t pad_cap)
{
	if (local_cap > c->local_cap) {
		if (c->d_local) cudaFree(c->d_local);
		c->d_local = nullptr; c->local_cap = 0;
		CUDA_TRY(cudaMalloc(&c->d_local, local_cap * sizeof(agb_record))); c->local_cap = local_cap;
	}
	if (pad_cap > c->pad_cap) {
		if (c->d_pad) cudaFree(c->d_pad);
		c->d_pad = nullptr; c->pad_cap = 0;
		CUDA_TRY(cudaMalloc(&c->d_pad, pad_cap * sizeof(agb_record))); c->pad_cap = pad_cap;
	}
	return AGB_OK;
}

/* the local part: this shard with its halos as one text, ownership by the cut rule.  first: nothing in front of the
 * shard (own range open to the left); open_end: nothing owned by anyone else behind it (own range open to the right);
 * reaches_end: the scanned bytes end where the whole text ends.
 * grow: a halo that is too short is not an error but a request for a longer one -- the result and part are filled and
 * the return value is HALO_SHORT_RIGHT and/or HALO_SHORT_LEFT (the windowed scan of scan.cu rescans with it doubled) */
static int shard_scan_geom(const agb_desc &d, const void *d_shard, uint64_t n_local, uint64_t halo_left, uint64_t halo_right,
                           bool first, bool open_end, bool reaches_end, int want, int want_level,
                           agb_record *d_records, uint64_t capacity, cudaStream_t st, agb_result *lres, agb_shard_part *part,
                           const agb_pattern *px = nullptr, bool grow = false, int dseed = -1, int64_t state_at = -1, int *state_out = nullptr)
{
	if (((uintptr_t)d_shard & 15) || (halo_left & 15)) { snprintf(g_err, sizeof g_err, "shard pointer and left halo must be 16-byte aligned"); return AGB_ERR_ARG; }
	if ((!first && (halo_left % 512)) || (!open_end && ((halo_left + n_local) % 512))) { snprintf(g_err, sizeof g_err, "shard boundaries must fall on multiples of 512 bytes of the scanned range"); return AGB_ERR_ARG; }
	const uint8_t *text = (const uint8_t *)d_shard - halo_left;
	const uint64_t n = halo_left + n_local + halo_right;
	ShardInfo sh;
	sh.own_lo = first ? INT64_MIN : (int64_t)halo_left;
	sh.own_hi = open_end ? INT64_MAX : (int64_t)(halo_left + n_local);
	sh.last = reaches_end ? 1 : 0;
	sh.dseed = dseed;
	int rc = scan_device_impl(d, text, n, want, want_level, d_records, (want & AGB_WANT_RECORDS) ? capacity : 0, st, lres, &sh, px);
	if (rc) return rc;
	memset(part, 0, sizeof *part);
	int dev = 0; CUDA_TRY(cudaGetDevice(&dev));
	/* the delimiter counts of the halos (ordinals) and the run check of the left halo came back with the scan's result
	 * (shard_aux_enqueue, launched by the scan before its one read-back) */
	std::lock_guard<std::mutex> lk(g_ws_mu[dev]);
	Workspace &W = g_ws[dev];
	const bool ord = (want & AGB_WANT_ORDINALS) != 0;
	if (state_out && d.delim_kind == 3 && state_at >= 0) {
		/* the delimiter's state at state_at (a multiple of 512) of the scanned range: where the next window's scan starts */
		uint8_t *h = reinterpret_cast<uint8_t *>(W.h_totals + 19);
		CUDA_TRY(cudaMemcpyAsync(h, W.dstate + state_at / 128, 1, cudaMemcpyDeviceToHost, st));
		CUDA_TRY(cudaStreamSynchronize(st));
		*state_out = *h;
	}
	const int short_halos = (W.h_totals[11] ? HALO_SHORT_RIGHT : 0) | (W.h_totals[18] ? HALO_SHORT_LEFT : 0);
	if (!grow && W.h_totals[11]) { snprintf(g_err, sizeof g_err, "a record of this shard runs past its halo (%d bytes behind the shard)", AGB_HALO_RIGHT); return AGB_ERR_ARG; }
	if (!grow && W.h_totals[18]) { snprintf(g_err, sizeof g_err, "a run of the delimiter longer than the left halo (%llu bytes) crosses the start of this shard", (unsigned long long)halo_left); return AGB_ERR_ARG; }
	part->byte_base = -(int64_t)halo_left;
	if (ord) {
		const unsigned long long total = lres->n_closes - (unsigned long long)W.ord_virt;     /* delimiter ends the local scan saw */
		const unsigned long long s_lo = W.h_totals[16], s_hi = open_end ? total : W.h_totals[17];
		part->closes = s_hi - s_lo;
		/* local ordinals count the local virtual '\n' and j0 correction, and the ends of the left halo */
		part->ord_fix = (long long)W.ord_virt + W.ord_j0 + (long long)s_lo;
		part->ord_origin = first ? (long long)W.ord_virt + W.ord_j0 : 0;
		part->virt = first ? W.ord_virt : 0;
	}
	return grow ? short_halos : AGB_OK;
}

/* one window of the windowed scan (scan.cu, scan_windowed): the shard scan in grow mode, then the window's records made
 * global on the device -- begin/end += byte_add, ordinal += ord_add -- by the gather kernel over a world of one */
int shard_window_scan(const agb_desc &d, const agb_pattern *px, const void *d_win, uint64_t n_local, uint64_t halo_left, uint64_t halo_right,
                      bool first, bool open_end, bool reaches_end, int want, agb_record *d_records, uint64_t capacity,
                      cudaStream_t st, agb_result *lres, agb_shard_part *part, int dseed, int64_t state_at, int *state_out)
{
	return shard_scan_geom(d, d_win, n_local, halo_left, halo_right, first, open_end, reaches_end, want, -1, d_records, capacity, st,
	                       lres, part, px, true, dseed, state_at, state_out);
}

/* the sharded scans cannot give a rank the delimiter's state at the start of its shard (the halos are too short for it) */
static int refuse_sticky(const agb_desc &d, char *err = nullptr, size_t errlen = 0)
{
	if (d.delim_kind != 3) return AGB_OK;
	const char *msg = "-p with a delimiter of more than one byte is not supported by the sharded scans (a shard's records depend on all the text before it)";
	snprintf(g_err, sizeof g_err, "%s", msg);
	if (err && errlen) snprintf(err, errlen, "%s", msg);
	return AGB_ERR_PATTERN;
}

int shard_window_rebase(agb_record *d_records, uint64_t n, long long byte_add, long long ord_add, bool ordinals, cudaStream_t st)
{
	if (!n) return AGB_OK;
	GatherParams G; memset(&G, 0, sizeof G);
	G.world = 1; G.pad = n; G.count[0] = n; G.out_off[0] = 0; G.byte_base[0] = byte_add; G.ord_add[0] = ord_add; G.ordinals = ordinals ? 1 : 0;
	dim3 grid((unsigned)std::min<uint64_t>((n + 255) / 256, 1024), 1);
	k_gather_compact<<<grid, 256, 0, st>>>(d_records, d_records, n, G); g_launches++;     /* in place: every thread reads, then writes, its own entry */
	CUDA_TRY(cudaGetLastError());
	return AGB_OK;
}

extern "C" int agb_scan_shard_local(const agb_pattern *p, const void *d_shard, uint64_t n_local, uint64_t halo_left, uint64_t halo_right,
                                    int first, int open_end, int reaches_end, int want, agb_record *d_records, uint64_t capacity,
                                    void *stream, agb_result *res, agb_shard_part *part)
{
	if (!p || !res || !part) return AGB_ERR_ARG;
	if ((want & AGB_WANT_RECORDS) && capacity && !d_records) return AGB_ERR_ARG;
	if (refuse_sticky(p->d)) return AGB_ERR_PATTERN;
	return shard_scan_geom(p->d, d_shard, n_local, halo_left, halo_right, first != 0, open_end != 0, reaches_end != 0, want, -1,
	                       d_records, capacity, (cudaStream_t)stream, res, part, p);
}

/* this rank's part of a sharded scan; fills its header */
static int shard_local_scan(const agb_desc &d, agb_comm *c, const void *d_shard, uint64_t n_local, int want, int want_level,
                            uint64_t local_cap, cudaStream_t st, agb_result *lres, const agb_pattern *px = nullptr)
{
	if (!c->halo_known || c->sizes[c->rank] != n_local) { snprintf(g_err, sizeof g_err, "agb_shard_halo() has not been called for this shard"); return AGB_ERR_ARG; }
	int rc = comm_buffers(c, (want & AGB_WANT_RECORDS) ? local_cap : 0, 0); if (rc) return rc;
	agb_shard_part part;
	rc = shard_scan_geom(d, d_shard, n_local, c->halo_left, c->halo_right, c->rank == 0, c->rank + 1 >= c->world, c->reaches_end != 0,
	                     want, want_level, c->d_local, local_cap, st, lres, &part, px);
	if (rc) return rc;
	unsigned long long *h = c->h_hdr;
	memset(h, 0, HDR_WORDS * sizeof *h);
	h[H_MATCHED] = lres->n_matched; h[H_RECORDS] = lres->n_records; h[H_FLAGGED] = lres->n_flagged;
	for (int l = 0; l <= AGB_MAXERR; l++) h[H_HIST + l] = lres->level_hist[l];
	h[H_TRUNC] = lres->truncated; h[H_NLOCAL] = n_local;
	float ms[2] = { lres->ms_front, lres->ms_records };
	memcpy(&h[H_MS_FRONT], &ms[0], sizeof(float)); memcpy(&h[H_MS_REC], &ms[1], sizeof(float));
	h[H_CLOSES] = part.closes; h[H_ORD_FIX] = (unsigned long long)part.ord_fix; h[H_ORD_ORIGIN] = (unsigned long long)part.ord_origin;
	h[H_VIRT] = (unsigned long long)part.virt;
	return AGB_OK;
}

/* headers of all ranks -> host (one synchronisation); sums into res */
static int shard_headers(agb_comm *c, cudaStream_t st, agb_result *res)
{
	CUDA_TRY(cudaMemcpyAsync(c->d_hdr, c->h_hdr, HDR_WORDS * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
	NCCL_TRY(ncclAllGather(c->d_hdr, c->d_all, HDR_WORDS, ncclUint64, c->nccl, st));
	CUDA_TRY(cudaMemcpyAsync(c->h_all, c->d_all, (size_t)c->world * HDR_WORDS * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
	CUDA_TRY(cudaStreamSynchronize(st));
	memset(res, 0, sizeof *res);
	float msf = 0, msr = 0;
	for (int r = 0; r < c->world; r++) {
		const unsigned long long *h = c->h_all + (size_t)r * HDR_WORDS;
		res->n_matched += h[H_MATCHED]; res->n_flagged += h[H_FLAGGED];
		for (int l = 0; l <= AGB_MAXERR; l++) res->level_hist[l] += h[H_HIST + l];
		res->n_closes += h[H_CLOSES];
		float a, b; memcpy(&a, &h[H_MS_FRONT], sizeof a); memcpy(&b, &h[H_MS_REC], sizeof b);
		msf = std::max(msf, a); msr = std::max(msr, b);
	}
	res->n_closes += c->h_all[H_VIRT];                              /* the virtual '\n' of the whole text */
	res->ms_front = msf; res->ms_records = msr;
	return AGB_OK;
}

/* the lists of all ranks (h_all[r][H_RECORDS] entries of c->d_local each) -> d_records on every rank */
static int shard_gather_lists(agb_comm *c, uint64_t global_offset, int want, agb_record *d_records, uint64_t capacity, cudaStream_t st, agb_result *res)
{
	GatherParams G; memset(&G, 0, sizeof G);
	G.world = c->world; G.ordinals = (want & AGB_WANT_ORDINALS) ? 1 : 0;
	uint64_t m = 0, total = 0; long long closes_before = (long long)c->h_all[H_ORD_ORIGIN]; uint64_t off = 0;
	bool trunc = false;
	for (int r = 0; r < c->world; r++) {
		const unsigned long long *h = c->h_all + (size_t)r * HDR_WORDS;
		G.count[r] = h[H_RECORDS]; G.out_off[r] = total; total += h[H_RECORDS];
		m = std::max<uint64_t>(m, h[H_RECORDS]);
		trunc = trunc || h[H_TRUNC] != 0;
		/* rank r's local scan starts AGB_HALO_LEFT bytes before its shard (rank 0: at its shard) */
		G.byte_base[r] = (long long)off - (r > 0 ? AGB_HALO_LEFT : 0);
		G.ord_add[r] = closes_before - (long long)h[H_ORD_FIX];
		closes_before += (long long)h[H_CLOSES];
		off += h[H_NLOCAL];
	}
	(void)global_offset;                                     /* (= the sum of the sizes before this rank: checked by the caller's layout) */
	res->n_records = std::min<uint64_t>(total, capacity);
	res->truncated = (trunc || total > capacity) ? 1 : 0;
	if (!m || !capacity) return AGB_OK;
	if (m > c->local_cap) return AGB_ERR_ARG;                       /* (every rank's list was cut to the capacity) */
	int rc = comm_buffers(c, 0, (uint64_t)c->world * m); if (rc) return rc;
	G.pad = m;
	NCCL_TRY(ncclAllGather(c->d_local, c->d_pad, m * sizeof(agb_record), ncclUint8, c->nccl, st));
	dim3 grid((unsigned)std::min<uint64_t>((m + 255) / 256, 1024), (unsigned)c->world);
	k_gather_compact<<<grid, 256, 0, st>>>(c->d_pad, d_records, capacity, G); g_launches++;
	CUDA_TRY(cudaGetLastError());
	CUDA_TRY(cudaStreamSynchronize(st));
	return AGB_OK;
}

extern "C" int agb_scan_sharded(const agb_pattern *p, agb_comm *c, const void *d_shard, uint64_t n_local, uint64_t global_offset,
                                int want, agb_record *d_records, uint64_t capacity, void *stream, agb_result *res)
{
	if (!p || !c || !res) return AGB_ERR_ARG;
	if ((want & AGB_WANT_RECORDS) && capacity && !d_records) return AGB_ERR_ARG;
	if (refuse_sticky(p->d)) return AGB_ERR_PATTERN;
	cudaStream_t st = (cudaStream_t)stream;
	CUDA_TRY(cudaSetDevice(c->dev));
	agb_result lres;
	/* a rank's own list can be as long as the whole capacity (all the matches may sit in one shard) */
	int rc = shard_local_scan(p->d, c, d_shard, n_local, want, -1, capacity, st, &lres, p); if (rc) return rc;
	rc = shard_headers(c, st, res); if (rc) return rc;
	if ((want & AGB_WANT_RECORDS) && capacity) { rc = shard_gather_lists(c, global_offset, want, d_records, capacity, st, res); if (rc) return rc; }
	return AGB_OK;
}

/* keep the records of one level (stable, in place): scan.cu */
__global__ void k_filter_level(agb_record *recs, uint64_t n, int level, unsigned long long *n_out);

extern "C" int agb_bestmatch_sharded(const char *pattern, const agb_options *opt, agb_comm *c, const void *d_shard, uint64_t n_local,
                                     uint64_t global_offset, agb_record *d_records, uint64_t capacity, void *stream,
                                     int *best_k, agb_result *res, char *err, size_t errlen)
{
	if (!pattern || !opt || !c || !best_k || !res) return AGB_ERR_ARG;
	if (capacity && !d_records) return AGB_ERR_ARG;
	cudaStream_t st = (cudaStream_t)stream;
	CUDA_TRY(cudaSetDevice(c->dev));
	agb_options o = *opt; agb_desc d; const int m = (int)strlen(pattern);
	o.bestmatch = 1; o.k = 0;
	*best_k = -1;
	int rc = agbi_build(pattern, &o, &d, err, errlen); if (rc) return rc;
	if (refuse_sticky(d, err, errlen)) return AGB_ERR_PATTERN;
	int kmax = d.M - 1; if (kmax > AGB_MAXERR) kmax = AGB_MAXERR; if (kmax > m - 1) kmax = m - 1;
	const int want = AGB_WANT_LEVELS | (capacity ? AGB_WANT_RECORDS : AGB_WANT_COUNT);
	const int stages[3] = { 2, 4, 8 }; int prev = -1;
	for (int si = 0; si < 3; si++) {
		const int k = stages[si] < kmax ? stages[si] : kmax;
		if (k <= prev) break;
		o.k = k;
		rc = agbi_build(pattern, &o, &d, err, errlen); if (rc) return rc;
		agb_result lres;
		rc = shard_local_scan(d, c, d_shard, n_local, want, -1, capacity, st, &lres); if (rc) return rc;
		rc = shard_headers(c, st, res); if (rc) return rc;          /* the histogram of the whole text: every rank sees the same */
		int best = -1;
		for (int l = prev + 1; l <= k; l++) if (res->level_hist[l]) { best = l; break; }
		prev = k;
		if (best < 0) continue;
		*best_k = best;
		const uint64_t n_best = res->level_hist[best];
		if (capacity) {
			/* every rank keeps its records of the best level of the WHOLE text, then the gather */
			bool any_trunc = false;
			for (int r = 0; r < c->world; r++) any_trunc = any_trunc || c->h_all[(size_t)r * HDR_WORDS + H_TRUNC] != 0;
			if (any_trunc) {
				o.k = best;
				rc = agbi_build(pattern, &o, &d, err, errlen); if (rc) return rc;
				rc = shard_local_scan(d, c, d_shard, n_local, want, best, capacity, st, &lres); if (rc) return rc;
			} else if (best < k && lres.n_records) {
				std::lock_guard<std::mutex> lk(g_ws_mu[c->dev]);
				Workspace &W = g_ws[c->dev];
				k_filter_level<<<1, 1024, 0, st>>>(c->d_local, lres.n_records, best, W.totals + 15); g_launches++;
				CUDA_TRY(cudaGetLastError());
				lres.n_records = std::min<uint64_t>(lres.level_hist[best], capacity);
				c->h_hdr[H_RECORDS] = lres.n_records;
			}
			if (any_trunc || best < k) {
				/* the list lengths changed: the headers once more */
				agb_result r2;
				rc = shard_headers(c, st, &r2); if (rc) return rc;
			}
			rc = shard_gather_lists(c, global_offset, want, d_records, capacity, st, res); if (rc) return rc;
		}
		res->n_matched = n_best;
		return AGB_OK;
	}
	res->n_matched = 0; res->n_records = 0;
	return AGB_OK;
}
