/*
 * client.c -- the runtime that libnvshare.so injects into a CUDA application:
 * registers with nvshare-scheduler, gates GPU work on the lock, and -- new in
 * this build -- drives the swap engine at every change of lock ownership.
 *
 * Behaviour kept from the reference (src/client.c), with its lines:
 *   - one REGISTER per process carrying pod name / namespace ("none" outside
 *     Kubernetes); the app blocks in its first cuInit / cuGetProcAddress until
 *     the scheduler has answered; no scheduler -> exit(1)        :180-204,213-294
 *   - continue_with_lock(): one REQ_LOCK per contention episode on behalf of
 *     all application threads, then wait for LOCK_OK               :73-106
 *   - DROP_LOCK: close the gate, drain the context, LOCK_RELEASED  :308-319
 *   - SCHED_OFF opens the gate for good, SCHED_ON closes it again  :320-340
 *   - idle detector: every 5 s, if no gated call happened and the GPU is idle
 *     (NVML utilisation 0, or a context sync shorter than 100 ms when NVML is
 *     unavailable) the lock is handed back voluntarily             :356-485
 *   - both library threads run with every signal blocked           :226-228
 *
 * What is new: the two data-path calls.
 *   LOCK_OK    -> datapath.fetch_all() BEFORE the gate opens.  VMM-backed
 *                 memory cannot page-fault, so the whole working set must be
 *                 mapped before any kernel of this process may run.
 *   DROP_LOCK / idle release / SCHED_ON -> after the context is drained,
 *                 datapath.evict(): HBM is released so the next holder can map
 *                 its own.  With NVSHARE_EARLY_RELEASE=1 (default)
 *                 LOCK_RELEASED is sent BEFORE evicting, so the next client's
 *                 fetch (host->HBM) overlaps our eviction (HBM->host) on the
 *                 full-duplex link; its cuMemCreate calls simply wait for the
 *                 HBM we are still releasing.
 *
 * The thread structure is the reference's (message thread + idle thread); the
 * state is one mutex and two condition variables.
 */
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <errno.h>
#include <inttypes.h>
#include <pthread.h>
#include <semaphore.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include "../../include/nvshare_wire.h"
#include "client.h"
#include "nvs_log.h"

#define IDLE_CHECK_SECONDS 5   /* reference src/client.c:51  */
#define IDLE_SYNC_BUSY_MS 100  /* reference src/client.c:466 */

static struct nvs_client_driver drv;
static struct nvs_client_datapath dp;
void (*nvs_client_on_context_sync)(void) = NULL;

static pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;
static pthread_cond_t lock_cv = PTHREAD_COND_INITIALIZER; /* own_lock became 1          */
static pthread_cond_t idle_cv = PTHREAD_COND_INITIALIZER; /* activity / lock hand-over  */
static pthread_cond_t drain_cv = PTHREAD_COND_INITIALIZER; /* inflight dropped to 0     */
static int inflight; /* application threads between the gate and the return of their driver call */
static int releasing; /* a release is in progress: REQ_LOCK must not overtake its LOCK_RELEASED     */
static sem_t registered;
static int sock_fd = -1;
static int scheduler_on, own_lock, need_lock, did_work;
static int nvml_ok;
static int early_release = 1;
static int sched_v2;          /* the daemon speaks the data-field hints (include/nvshare_wire.h)   */
static int evict_all_policy;  /* NVSHARE_EVICT_POLICY=all: never keep slabs resident without lock */
static pthread_mutex_t send_mu = PTHREAD_MUTEX_INITIALIZER; /* frames from several threads      */
/* head-room left free beyond what the next client asked for: 1/512 of the HBM, 16 MiB..1 GiB */
static uint64_t evict_margin_mib(void);
static uint64_t client_id;
static CUcontext app_ctx;
static int app_ctx_known;

static void block_all_signals(void)
{
	sigset_t all;
	nvs_must(sigfillset(&all) == 0);
	nvs_must(pthread_sigmask(SIG_SETMASK, &all, NULL) == 0);
}

static void send_msg(uint8_t type, const char *hint)
{
	struct nvs_msg m;
	memset(&m, 0, sizeof(m));
	m.type = type;
	m.id = client_id;
	if (hint)
		snprintf(m.data, sizeof(m.data), "%s", hint);
	pthread_mutex_lock(&send_mu);
	ssize_t w = nvs_write_all(sock_fd, &m, sizeof(m));
	pthread_mutex_unlock(&send_mu);
	nvs_must(w == (ssize_t)sizeof(m));
	nvs_debug("Sent %s %s", nvs_msg_type_name(type), hint ? hint : "");
}

/* Drain everything the application has submitted (mutex held). */
static void sync_app_context(void)
{
	if (nvs_client_on_context_sync)
		nvs_client_on_context_sync();
	if (!app_ctx_known)
		return; /* the app never issued gated work: nothing can be in flight */
	CUresult r = drv.cuCtxSetCurrent(app_ctx);
	if (r != CUDA_SUCCESS)
		nvs_warn("cuCtxSetCurrent returned %d", (int)r);
	r = drv.cuCtxSynchronize();
	if (r != CUDA_SUCCESS)
		nvs_warn("cuCtxSynchronize returned %d", (int)r);
}

static void close_gate_and_drain(void);

static void set_own_lock(int v)
{
	own_lock = v;
	if (dp.lock_state)
		dp.lock_state(v);
}

void nvs_client_pressure(uint64_t mib)
{
	char hint[NVS_MSG_DATA_LEN];
	if (sock_fd < 0 || !sched_v2)
		return; /* the reference daemon would take it for a plain lock request (and nobody is lazily resident under it) */
	snprintf(hint, sizeof(hint), "%c%" PRIu64, NVS_HINT_PRESSURE_PREFIX, mib);
	send_msg(NVS_REQ_LOCK, hint);
}

#define EVICT_ALL UINT64_MAX
#define FAVOUR_MIN_MIB 8192 /* smallest eviction done on a pressure hint */

static uint64_t evict_margin_mib(void)
{
	/* 1/512 of the HBM (160 MiB on an 80 GB H100): covers the 64 MiB of slack the fetching side wants to
	 * see free beyond what it maps (engine.c wait_for_hbm_burst) and the context growth of a client
	 * that starts using a library between two hand-offs.  Every MiB of it crosses the link twice per
	 * hand-off for nothing, hence no more than that (round 1 used 1/128: 1.5 GiB). */
	uint64_t total = dp.total_hbm_mib ? dp.total_hbm_mib() : 0;
	uint64_t m = total / 512;
	return m < 16 ? 16 : m > 1024 ? 1024 : m;
}

/*
 * How much HBM to give up when the lock leaves us.
 *   - daemon without hints (the reference's), or NVSHARE_EVICT_POLICY=all: everything.
 *     A client without the lock then holds no swappable HBM -- always safe.
 *   - nobody is waiting (waiters == 0, or an idle release): nothing.  If someone
 *     needs the memory later, the daemon forwards its pressure ("e<MiB>").
 *   - otherwise just enough for the next client's stated need plus head-room.
 */
static uint64_t eviction_amount_mib(int have_hint, unsigned waiters, uint64_t need_mib)
{
	if (!sched_v2 || evict_all_policy)
		return EVICT_ALL;
	if (!have_hint || waiters == 0)
		return 0;
	uint64_t want = need_mib + evict_margin_mib();
	uint64_t free_mib = dp.free_hbm_mib ? dp.free_hbm_mib() : 0;
	return want > free_mib ? want - free_mib : 0;
}

static void do_evict(uint64_t mib)
{
	if (!dp.evict || mib == 0)
		return;
	if (dp.evict(mib == EVICT_ALL ? 0 : mib << 20) != 0)
		nvs_fatal("eviction failed; cannot hand the GPU over safely");
}

/* An eviction done as a favour (memory pressure from the client that is mapping).  It
 * must not wait for room in the backing pool: our own LOCK_OK may be queued right behind
 * this message, and the fetch it triggers is what would free that room. */
static void do_evict_as_a_favour(uint64_t mib)
{
	if (!dp.evict_best_effort) {
		do_evict(mib);
		return;
	}
	if (mib != 0 && dp.evict_best_effort(mib == EVICT_ALL ? 0 : mib << 20) != 0)
		nvs_fatal("eviction failed; cannot hand the GPU over safely");
}

/* Give the lock back and get our slabs out of the next holder's way (mutex held). */
static void release_lock_and_evict(int have_hint, unsigned waiters, uint64_t need_mib)
{
	releasing = 1;
	close_gate_and_drain();
	sync_app_context();
	uint64_t mib = eviction_amount_mib(have_hint, waiters, need_mib);
	if (mib != 0 && dp.evict_announce)
		dp.evict_announce(); /* before the next holder is told to go: its fetch then follows our progress */
	if (early_release)
		send_msg(NVS_LOCK_RELEASED, NULL);
	do_evict(mib);
	if (!early_release)
		send_msg(NVS_LOCK_RELEASED, NULL);
	releasing = 0;
	/* threads parked at the gate may now ask for the lock again (behind the waiters) */
	nvs_must(pthread_cond_broadcast(&lock_cv) == 0);
}

void continue_with_lock(void)
{
	nvs_must(pthread_mutex_lock(&mu) == 0);
	if (!app_ctx_known) {
		CUcontext c = NULL;
		if (drv.cuCtxGetCurrent(&c) != CUDA_SUCCESS)
			nvs_fatal("Can't get app's CUDA context!");
		if (c != NULL) { /* a launch without a context fails in the driver anyway */
			app_ctx = c;
			app_ctx_known = 1;
		}
	}
	while (!own_lock) {
		if (!need_lock && !releasing) { /* one request on behalf of every application thread */
			char hint[NVS_MSG_DATA_LEN];
			need_lock = 1;
			snprintf(hint, sizeof(hint), "%c%" PRIu64, NVS_HINT_NEED_PREFIX,
				 dp.nonresident_mib ? dp.nonresident_mib() : 0);
			send_msg(NVS_REQ_LOCK, hint);
		}
		nvs_must(pthread_cond_wait(&lock_cv, &mu) == 0);
	}
	did_work = 1;
	inflight++; /* paired with nvs_gate_leave() once the driver call has been issued */
	nvs_must(pthread_cond_broadcast(&idle_cv) == 0);
	nvs_must(pthread_mutex_unlock(&mu) == 0);
}

void nvs_gate_leave(void)
{
	nvs_must(pthread_mutex_lock(&mu) == 0);
	if (--inflight == 0)
		nvs_must(pthread_cond_broadcast(&drain_cv) == 0);
	nvs_must(pthread_mutex_unlock(&mu) == 0);
}

/*
 * Close the gate and wait until every application thread that had already passed
 * it has handed its call to the driver.  The reference only clears own_lock
 * (src/client.c:312): with managed memory a late launch merely faults pages back
 * in; with VMM memory it would touch slabs that are being unmapped.  Mutex held.
 */
static void close_gate_and_drain(void)
{
	set_own_lock(0);
	while (inflight > 0)
		nvs_must(pthread_cond_wait(&drain_cv, &mu) == 0);
}

static void fill_identity(struct nvs_msg *m)
{
	const char *ns_file = "/var/run/secrets/kubernetes.io/serviceaccount/namespace";
	snprintf(m->pod_name, sizeof(m->pod_name), "none");
	snprintf(m->pod_namespace, sizeof(m->pod_namespace), "none");
	if (!getenv("KUBERNETES_SERVICE_HOST"))
		return;
	FILE *f = fopen(ns_file, "r");
	if (!f || !fgets(m->pod_namespace, sizeof(m->pod_namespace), f)) {
		nvs_warn("Couldn't read the Pod namespace from %s", ns_file);
		snprintf(m->pod_namespace, sizeof(m->pod_namespace), "none");
	}
	if (f)
		fclose(f);
	const char *host = getenv("HOSTNAME");
	if (host) {
		if (strlen(host) >= sizeof(m->pod_name))
			nvs_warn("Pod name is longer than %zu characters. Truncating it.", sizeof(m->pod_name));
		snprintf(m->pod_name, sizeof(m->pod_name), "%s", host);
	}
}

static void *message_thread(void *arg)
{
	(void)arg;
	struct nvs_msg in, out;
	char path[108];

	block_all_signals();
	if (drv.cuInit(0) != CUDA_SUCCESS)
		nvs_fatal("cuInit failed when initializing client");

	memset(&out, 0, sizeof(out));
	out.type = NVS_REGISTER;
	out.id = NVS_ID_CLIENT_PREREG;
	snprintf(out.data, sizeof(out.data), "nvs2"); /* the reference daemon ignores REGISTER.data */
	fill_identity(&out);
	nvs_debug("NVSHARE_POD_NAME = %s", out.pod_name);
	nvs_debug("NVSHARE_POD_NAMESPACE = %s", out.pod_namespace);

	nvs_must(nvs_socket_path(path, sizeof(path)) == 0);
	if ((sock_fd = nvs_connect(path)) < 0) {
		nvs_info("Failed to connect to UNIX socket at %s\n", path);
		nvs_fatal("Condition failed: nvshare_connect(&rsock, nvscheduler_socket_path) == 0");
	}
	nvs_must(nvs_write_all(sock_fd, &out, sizeof(out)) == (ssize_t)sizeof(out));
	nvs_debug("Sent %s", nvs_msg_type_name(out.type));

	memset(&in, 0, sizeof(in));
	nvs_must(nvs_read_all(sock_fd, &in, sizeof(in)) == (ssize_t)sizeof(in));
	if (in.type != NVS_SCHED_ON && in.type != NVS_SCHED_OFF)
		nvs_fatal("Got message with type (%d) instead of initial nvshare-scheduler status", (int)in.type);
	nvs_debug("Received %s", nvs_msg_type_name(in.type));
	sched_v2 = (in.data[17] == NVS_CAP_MARKER);
	in.data[16] = '\0';
	unsigned long long id = 0;
	nvs_must(sscanf(in.data, "%llx", &id) == 1);
	client_id = id;
	nvs_info("Successfully initialized nvshare GPU");
	nvs_info("Client ID = %016" PRIx64, client_id);
	scheduler_on = (in.type == NVS_SCHED_ON);
	need_lock = 0;
	set_own_lock(!scheduler_on);
	nvs_must(sem_post(&registered) == 0);

	for (;;) {
		memset(&in, 0, sizeof(in));
		nvs_must(nvs_read_all(sock_fd, &in, sizeof(in)) == (ssize_t)sizeof(in));
		nvs_must(pthread_mutex_lock(&mu) == 0);
		switch (in.type) {
		case NVS_LOCK_OK:
			nvs_debug("Received %s", nvs_msg_type_name(in.type));
			/* VMM memory cannot fault: be fully resident before the gate opens */
			if (dp.fetch_all && dp.fetch_all() != 0)
				nvs_fatal("could not make the working set resident after LOCK_OK");
			need_lock = 0;
			set_own_lock(1);
			did_work = 1; /* restart the idle timer */
			nvs_must(pthread_cond_broadcast(&lock_cv) == 0);
			nvs_must(pthread_cond_broadcast(&idle_cv) == 0);
			break;
		case NVS_DROP_LOCK: {
			in.data[NVS_MSG_DATA_LEN - 1] = '\0';
			nvs_debug("Received %s %s", nvs_msg_type_name(in.type), in.data);
			if (in.data[0] == NVS_HINT_EVICT_PREFIX) {
				/* Memory pressure forwarded by the daemon: never a quantum expiry, whoever holds the
				 * lock.  A frame queued while we were busy (a long fetch) may only be looked at once
				 * we are the holder: it is stale then -- the client that pressed has since released,
				 * or is waiting behind us and will be served when our quantum ends. */
				if (own_lock) {
					nvs_debug("pressure hint reached the lock holder: ignored");
					break;
				}
				/* the client that is mapping is short of HBM: get out of its way */
				uint64_t mib = strtoull(in.data + 1, NULL, 10);
				sync_app_context();
				/* At least FAVOUR_MIN_MIB at a time: a framework that is building its state allocates
				 * thousands of blocks, each of which stalls before it presses (a ResNet-50 client
				 * took minutes to set up beside an idle one that gave way 1 GiB at a time).  We do not
				 * hold the lock: whatever goes now comes back with our next fetch. */
				if (mib && mib < FAVOUR_MIN_MIB)
					mib = FAVOUR_MIN_MIB;
				do_evict_as_a_favour(mib ? mib + evict_margin_mib() : EVICT_ALL);
				if (need_lock) {
					/* our queued request still advertises the old need: refresh it, or the
					 * holder will free too little for us and we will have to press it again */
					char hint[NVS_MSG_DATA_LEN];
					snprintf(hint, sizeof(hint), "%c%" PRIu64, NVS_HINT_NEED_PREFIX,
						 dp.nonresident_mib ? dp.nonresident_mib() : 0);
					send_msg(NVS_REQ_LOCK, hint);
				}
			} else if (own_lock && scheduler_on) {
				unsigned waiters = 0;
				unsigned long long need = 0;
				int have = sscanf(in.data, "w%un%llu", &waiters, &need) == 2;
				release_lock_and_evict(have, waiters, need);
			}
			break;
		}
		case NVS_SCHED_ON:
			nvs_debug("Received %s", nvs_msg_type_name(in.type));
			if (!scheduler_on) {
				nvs_debug("Scheduler status changed to ON");
				scheduler_on = 1;
				need_lock = 0;
				/* we were running ungated: stop, drain, and (unless the daemon will
				 * tell us when somebody needs the memory) get out of HBM */
				close_gate_and_drain();
				sync_app_context();
				do_evict(eviction_amount_mib(0, 0, 0));
			} else {
				nvs_debug("Scheduler status did not change, doing nothing");
			}
			break;
		case NVS_SCHED_OFF:
			nvs_debug("Received %s", nvs_msg_type_name(in.type));
			if (scheduler_on) {
				nvs_debug("Scheduler status changed to OFF");
				scheduler_on = 0;
				need_lock = 0;
				/* every client now runs at once: only possible if all of us fit */
				if (dp.fetch_all && dp.fetch_all() != 0)
					nvs_fatal("anti-thrashing was turned off but the working sets do not fit in HBM");
				set_own_lock(1);
				nvs_must(pthread_cond_broadcast(&lock_cv) == 0);
			}
			break;
		default:
			nvs_warn("Unknown message type (%d)", (int)in.type);
			break;
		}
		nvs_must(pthread_mutex_unlock(&mu) == 0);
	}
	return NULL;
}

/* The NVML handle of the GPU the application's context is on (mutex held, context known).  NVML numbers
 * the physical GPUs whatever CUDA_VISIBLE_DEVICES says, so the driver is asked for the device's UUID and NVML
 * for the handle of that UUID.  Returns 0 and leaves *dev alone when any link of that chain is missing: the
 * caller then stays with index 0, the reference's choice. */
static int nvml_device_of_app(nvmlDevice_t *dev)
{
	CUdevice d = 0;
	uint8_t u[16];
	char name[48];
	nvmlDevice_t h = NULL;
	if (!drv.nvmlDeviceGetHandleByUUID || !drv.cuCtxGetDevice || !drv.cuDeviceGetUuid || !app_ctx_known)
		return 0;
	if (drv.cuCtxSetCurrent(app_ctx) != CUDA_SUCCESS || drv.cuCtxGetDevice(&d) != CUDA_SUCCESS ||
	    drv.cuDeviceGetUuid(u, d) != CUDA_SUCCESS)
		return 0;
	snprintf(name, sizeof(name), "GPU-%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", u[0], u[1], u[2],
		 u[3], u[4], u[5], u[6], u[7], u[8], u[9], u[10], u[11], u[12], u[13], u[14], u[15]);
	if (drv.nvmlDeviceGetHandleByUUID(name, &h) != NVML_SUCCESS || !h) {
		nvs_debug("NVML does not know %s (CUDA device %d): watching NVML device 0 like the reference", name, (int)d);
		return 0;
	}
	nvs_debug("Early release watches the utilisation of %s (CUDA device %d)", name, (int)d);
	*dev = h;
	return 1;
}

static void *idle_thread(void *arg)
{
	(void)arg;
	nvmlDevice_t nvml_dev = NULL;
	int nvml_dev_settled = 0; /* the application's own GPU has been looked up (it has no context before its first gated call) */
	block_all_signals();
	if (nvml_ok) {
		/* device index 0, like the reference (src/client.c:386), until the application's GPU is known */
		if (drv.nvmlInit() != NVML_SUCCESS || drv.nvmlDeviceGetHandleByIndex(0, &nvml_dev) != NVML_SUCCESS) {
			nvs_warn("NVML initialisation failed; falling back to timing cuCtxSynchronize");
			nvml_ok = 0;
		}
	}
	nvs_must(pthread_mutex_lock(&mu) == 0);
	for (;;) {
		struct timespec until;
		did_work = 0;
		nvs_must(clock_gettime(CLOCK_REALTIME, &until) == 0);
		until.tv_sec += IDLE_CHECK_SECONDS;
		int rc;
		do {
			rc = pthread_cond_timedwait(&idle_cv, &mu, &until);
		} while (rc == 0 && !did_work); /* spurious wake-up: keep waiting out the interval */
		if (rc == 0)
			continue; /* activity: restart the interval */
		if (rc != ETIMEDOUT) {
			errno = rc;
			nvs_fatal_errno("pthread_cond_timedwait() failed");
		}
		if (!scheduler_on || !own_lock || did_work)
			continue;
		/* nothing was submitted for a whole interval; is the GPU still busy with earlier work? */
		if (nvml_ok && !nvml_dev_settled && app_ctx_known) {
			nvml_device_of_app(&nvml_dev);
			nvml_dev_settled = 1;
		}
		if (nvml_ok) {
			nvmlUtilization_t u;
			if (drv.nvmlDeviceGetUtilizationRates(nvml_dev, &u) != NVML_SUCCESS) {
				nvs_warn("nvmlDeviceGetUtilizationRates failed; not using NVML any more");
				nvml_ok = 0;
				continue;
			}
			nvs_debug("GPU Utilization = %u %%", u.gpu);
			if (u.gpu > 0) {
				nvs_debug("Early release timer elapsed but we are not idle");
				continue;
			}
		} else {
			struct timespec a, b;
			clock_gettime(CLOCK_MONOTONIC, &a);
			sync_app_context();
			clock_gettime(CLOCK_MONOTONIC, &b);
			long ms = (b.tv_sec - a.tv_sec) * 1000 + (b.tv_nsec - a.tv_nsec) / 1000000;
			if (ms >= IDLE_SYNC_BUSY_MS) {
				nvs_debug("Early release timer elapsed but we are not idle");
				continue;
			}
		}
		nvs_debug("Releasing the lock early due to inactivity");
		release_lock_and_evict(0, 0, 0);
	}
	return NULL;
}

void nvs_client_start(const struct nvs_client_driver *d, const struct nvs_client_datapath *datapath)
{
	pthread_t t;
	drv = *d;
	if (datapath)
		dp = *datapath;
	nvml_ok = drv.nvmlInit && drv.nvmlDeviceGetHandleByIndex && drv.nvmlDeviceGetUtilizationRates;
	const char *er = getenv("NVSHARE_EARLY_RELEASE");
	if (er && *er)
		early_release = atoi(er) != 0;
	const char *pol = getenv("NVSHARE_EVICT_POLICY");
	evict_all_policy = pol && strcmp(pol, "all") == 0;
	nvs_must(sem_init(&registered, 0, 0) == 0);
	nvs_must(pthread_create(&t, NULL, message_thread, NULL) == 0);
	/* the application does not proceed until the scheduler has told us its status */
	int rc;
	do {
		rc = sem_wait(&registered);
	} while (rc != 0 && errno == EINTR);
	nvs_must(rc == 0);
	nvs_must(pthread_create(&t, NULL, idle_thread, NULL) == 0);
}
