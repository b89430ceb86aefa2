# ORACLE build (test infrastructure): the wildcard-minimization oracle.  Output: oracle/liboracle_wildcard.so
# (git-ignored).  The same sources as liboracle.so (Makefile), with sts.c replaced by sts_wildcard.c, which includes
# it and adds the WildCardMatch replay, plus the clusterizer and minimizer loop of wildcard.c.
CC ?= gcc
CFLAGS ?= -O3 -march=native -fPIC -Wall -Wextra -std=gnu11 -pthread
SRCS := machine.c models.c model_ir.c fuzz.c ddmin.c dpor.c dpor_frontier.c intmin.c provenance.c sts_wildcard.c wildcard.c
liboracle_wildcard.so: $(SRCS) sts.c sts.h sts_wildcard.h machine.h jrandom.h ../include/demi_b200.h ../include/demi_limits.h ../include/demi_model_ir.h
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS)
clean:
	rm -f liboracle_wildcard.so
