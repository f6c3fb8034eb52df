/* An LD_PRELOAD interposer on cudaFuncSetAttribute that holds open the window between one thread's set of a kernel's
 * dynamic shared-memory limit and its launch, so that tests can put another thread's set into that window on purpose.
 *
 * Every call is forwarded to the CUDA runtime's own cudaFuncSetAttribute first (cudaErrorUnknown when the process has
 * not loaded a runtime).  Once gate_arm(min_bytes, timeout_ms) has been called,
 * the first cudaFuncAttributeMaxDynamicSharedMemorySize set of at least min_bytes then holds its thread until another
 * thread sets the same kernel's limit (a release) or timeout_ms passes (a timeout), and disarms the gate.  Nothing waits
 * on the device, and every wait has a timeout. */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <errno.h>
#include <pthread.h>
#include <stddef.h>
#include <time.h>

enum { kMaxDynamicSmem = 8, kErrorUnknown = 999 };   /* cudaFuncAttributeMaxDynamicSharedMemorySize, cudaErrorUnknown */

typedef int (*set_attr_fn)(const void*, int, int);

static pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;
static pthread_cond_t cv = PTHREAD_COND_INITIALIZER;
static int armed_min;          /* > 0: the next set of at least this many bytes is held */
static int armed_timeout_ms;
static const void* held;       /* the kernel whose set is being held, NULL when none */
static int released;           /* the current hold was ended by another thread */
static int holds, releases, timeouts;

static void deadline_after(struct timespec* t, int ms)
{
    clock_gettime(CLOCK_REALTIME, t);
    t->tv_sec += ms / 1000;
    t->tv_nsec += (long)(ms % 1000) * 1000000L;
    if (t->tv_nsec >= 1000000000L) { t->tv_sec += 1; t->tv_nsec -= 1000000000L; }
}

/* The runtime's own function.  A library that links the runtime and is loaded with dlopen (ctypes.CDLL) brings it in
 * outside the global scope, where RTLD_NEXT does not look, so the runtime already loaded is also asked by name.  Nothing
 * is loaded here. */
static set_attr_fn real_set_attr(void)
{
    static const char* const names[] = {"libcudart.so.12", "libcudart.so"};
    void* f = dlsym(RTLD_NEXT, "cudaFuncSetAttribute");
    for (size_t i = 0; !f && i < sizeof(names) / sizeof(names[0]); ++i) {
        void* h = dlopen(names[i], RTLD_LAZY | RTLD_NOLOAD);
        if (h) {
            f = dlsym(h, "cudaFuncSetAttribute");
            dlclose(h);
        }
    }
    return (set_attr_fn)f;
}

int cudaFuncSetAttribute(const void* func, int attr, int value)
{
    const set_attr_fn real = real_set_attr();
    const int rc = real ? real(func, attr, value) : kErrorUnknown;
    if (attr != kMaxDynamicSmem) return rc;
    pthread_mutex_lock(&mu);
    if (held && func == held) {            /* the holder waits below, so this set comes from another thread */
        released = 1;
        ++releases;
        pthread_cond_broadcast(&cv);
    } else if (!held && armed_min > 0 && value >= armed_min) {
        struct timespec until;
        deadline_after(&until, armed_timeout_ms);
        armed_min = 0;
        held = func;
        released = 0;
        ++holds;
        pthread_cond_broadcast(&cv);       /* gate_wait_held */
        while (!released)
            if (pthread_cond_timedwait(&cv, &mu, &until) == ETIMEDOUT) { ++timeouts; break; }
        held = NULL;
    }
    pthread_mutex_unlock(&mu);
    return rc;
}

/* Hold the next limit set of at least min_bytes for at most timeout_ms. */
void gate_arm(int min_bytes, int timeout_ms)
{
    pthread_mutex_lock(&mu);
    armed_min = min_bytes;
    armed_timeout_ms = timeout_ms;
    pthread_mutex_unlock(&mu);
}

/* -> 1 once the armed hold has begun (it may have ended since), 0 if it has not within timeout_ms */
int gate_wait_held(int timeout_ms)
{
    struct timespec until;
    int ok = 1;
    deadline_after(&until, timeout_ms);
    pthread_mutex_lock(&mu);
    while (armed_min > 0)
        if (pthread_cond_timedwait(&cv, &mu, &until) == ETIMEDOUT) { ok = armed_min == 0; break; }
    pthread_mutex_unlock(&mu);
    return ok;
}

/* -> 1 when calls reach a CUDA runtime, 0 when they return cudaErrorUnknown for want of one */
int gate_forwards(void)
{
    return real_set_attr() != NULL;
}

/* Holds begun, holds ended by another thread's set, and holds ended by their timeout, since the library was loaded. */
void gate_stats(int* n_holds, int* n_releases, int* n_timeouts)
{
    pthread_mutex_lock(&mu);
    *n_holds = holds;
    *n_releases = releases;
    *n_timeouts = timeouts;
    pthread_mutex_unlock(&mu);
}
