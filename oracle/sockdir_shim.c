/*
 * sockdir_shim.c -- TEST INFRASTRUCTURE ONLY (never part of the product).
 *
 * The reference's daemon, CLI and library only know one socket directory,
 * /var/run/nvshare/ (src/comm.h:45), which an ordinary user can neither create
 * nor write.  Preloaded into the UNMODIFIED reference binaries, this library
 * gives them the knob ours has: when NVSHARE_SOCK_DIR is set, every path under
 * /var/run/nvshare that the reference passes to mkdir, chmod, unlink, bind or
 * connect is taken under that directory instead.  Without NVSHARE_SOCK_DIR it
 * changes nothing.  What the reference prints keeps its own path.
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <errno.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/types.h>
#include <sys/un.h>
#include <unistd.h>

#define REF_DIR "/var/run/nvshare"

/* out <- NVSHARE_SOCK_DIR + the part of `path` after /var/run/nvshare; 0 when nothing is redirected */
static int redirect(const char *path, char *out, size_t len)
{
	const char *dir = getenv("NVSHARE_SOCK_DIR");
	size_t n = strlen(REF_DIR);
	if (!dir || !*dir || !path || strncmp(path, REF_DIR, n) != 0 || (path[n] != '\0' && path[n] != '/'))
		return 0;
	size_t d = strlen(dir);
	while (d > 1 && dir[d - 1] == '/')
		--d;
	if ((size_t)snprintf(out, len, "%.*s%s", (int)d, dir, path + n) >= len)
		return -1;
	return 1;
}

typedef int (*path_fn)(const char *, mode_t);
typedef int (*unlink_fn)(const char *);
typedef int (*addr_fn)(int, const struct sockaddr *, socklen_t);
#define REAL(name, type) static type real_##name; if (!real_##name) real_##name = (type)dlsym(RTLD_NEXT, #name)

int mkdir(const char *path, mode_t mode)
{
	REAL(mkdir, path_fn);
	char buf[4096];
	int r = redirect(path, buf, sizeof(buf));
	if (r < 0)
		return errno = ENAMETOOLONG, -1;
	return real_mkdir(r ? buf : path, mode);
}

int chmod(const char *path, mode_t mode)
{
	REAL(chmod, path_fn);
	char buf[4096];
	int r = redirect(path, buf, sizeof(buf));
	if (r < 0)
		return errno = ENAMETOOLONG, -1;
	return real_chmod(r ? buf : path, mode);
}

int unlink(const char *path)
{
	REAL(unlink, unlink_fn);
	char buf[4096];
	int r = redirect(path, buf, sizeof(buf));
	if (r < 0)
		return errno = ENAMETOOLONG, -1;
	return real_unlink(r ? buf : path);
}

/* a sockaddr_un under /var/run/nvshare -> the same name under NVSHARE_SOCK_DIR; 0 when not redirected */
static int redirect_addr(const struct sockaddr *addr, socklen_t len, struct sockaddr_un *out)
{
	if (!addr || addr->sa_family != AF_UNIX || len <= offsetof(struct sockaddr_un, sun_path))
		return 0;
	const struct sockaddr_un *un = (const struct sockaddr_un *)addr;
	char path[sizeof(un->sun_path) + 1];
	size_t n = len - offsetof(struct sockaddr_un, sun_path);
	if (n > sizeof(un->sun_path))
		n = sizeof(un->sun_path);
	memcpy(path, un->sun_path, n);
	path[n] = '\0';
	memset(out, 0, sizeof(*out));
	out->sun_family = AF_UNIX;
	return redirect(path, out->sun_path, sizeof(out->sun_path));
}

int bind(int fd, const struct sockaddr *addr, socklen_t len)
{
	REAL(bind, addr_fn);
	struct sockaddr_un un;
	int r = redirect_addr(addr, len, &un);
	if (r < 0)
		return errno = ENAMETOOLONG, -1;
	return r ? real_bind(fd, (struct sockaddr *)&un, sizeof(un)) : real_bind(fd, addr, len);
}

int connect(int fd, const struct sockaddr *addr, socklen_t len)
{
	REAL(connect, addr_fn);
	struct sockaddr_un un;
	int r = redirect_addr(addr, len, &un);
	if (r < 0)
		return errno = ENAMETOOLONG, -1;
	return r ? real_connect(fd, (struct sockaddr *)&un, sizeof(un)) : real_connect(fd, addr, len);
}
