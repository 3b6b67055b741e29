/* tests/oracle_bfs.c -- TEST INFRASTRUCTURE ONLY.  The C restatement's BKTree::InitSearchTrees with EnableBfs
 * (BKT/ParameterDefinitionList.h:12, BKTree.h:696-769 incl. the m_bfs != 0 branch at :703-758).
 *
 * Not compiled on its own: tests/oracle_bfs.py appends it to an unchanged copy of oracle/sptag_oracle.c whose
 * bkt_init_search_trees is renamed bkt_init_search_trees_default, so that every search path of the pinned restatement
 * (search, RefineSearchIndex, ResultIterator, SearchIndexIterativeFromNeareast) seeds its trees through the function
 * below.  EnableBfs is a process-wide value, ora_set_bfs; an iterator reads it at its first call, where the reference's
 * InitSearchTrees runs. */

static int32_t g_bfs; /* BKTree::m_bfs */

void ora_set_bfs(int32_t bfs) { g_bfs = bfs; }

enum { kBfsMaxNodes = 100 }; /* MaxBFSNodes (BKTree.h:705) */

/* The children of node `tn` in child order: into the BFS heap `q` while dist <= 1.1f * q->Top() (an fp32 product; Top()
 * of the empty heap is the 1e9 the reference writes into heap[0]) and q holds fewer than MaxBFSNodes, into SPTQueue
 * otherwise */
static void bkt_bfs_admit(const qctx_t* c, ws_t* ws, heap_t* q, const ora_bkt_node* tn)
{
    const ora_bkt_node* nodes = (const ora_bkt_node*)c->idx->nodes;
    for (int32_t begin = tn->childStart; begin < tn->childEnd; begin++) {
        ws->ntree++;
        pair_t p = {begin, qdist(c, ws, nodes[begin].centerid)};
        const float top = q->count == 0 ? 1e9f : q->heap[1].distance;
        if (p.distance <= 1.1f * top && q->count < kBfsMaxNodes)
            heap_insert(q, p);
        else
            heap_insert(&ws->spt, p);
    }
}

/* One tree whose root has children (BKTree.h:703-758).  m_currBSPTQueue / m_nextBSPTQueue are Resize(MaxBFSNodes)d for
 * every tree.  A popped leaf goes to SPTQueue (no CheckAndSet, not counted); a popped internal node's centre enters
 * NGQueue if new (not a checked leaf) and its children are admitted to `next`.  Levels after the one that left `curr`
 * empty do nothing, so the loop stops there (the reference runs all m_bfs).  Negative values run no level. */
static void bkt_init_search_trees_bfs(const qctx_t* c, ws_t* ws, const ora_bkt_node* root)
{
    const ora_bkt_node* nodes = (const ora_bkt_node*)c->idx->nodes;
    pair_t a[kBfsMaxNodes + 1], b[kBfsMaxNodes + 1];
    heap_t ha = {a, kBfsMaxNodes, 0, 64}, hb = {b, kBfsMaxNodes, 0, 64}; /* admission never fills them */
    heap_t* curr = &ha;
    heap_t* next = &hb;
    bkt_bfs_admit(c, ws, curr, root);
    for (int32_t level = 1; level <= g_bfs && curr->count != 0; level++) {
        while (curr->count != 0) {
            pair_t tmp = heap_pop(curr);
            const ora_bkt_node* tnode = &nodes[tmp.node];
            ws->ntree++;
            if (tnode->childStart < 0) {
                heap_insert(&ws->spt, tmp);
            } else {
                if (!ws_check_and_set(ws, tnode->centerid)) {
                    pair_t p = {tnode->centerid, tmp.distance};
                    heap_insert(&ws->ng, p);
                }
                bkt_bfs_admit(c, ws, next, tnode);
            }
        }
        heap_t* t = curr;
        curr = next;
        next = t;
    }
    while (curr->count != 0) heap_insert(&ws->spt, heap_pop(curr));
}

/* BKTree::InitSearchTrees (BKTree.h:696-769); m_bfs == 0 is the restatement's own default seeding */
static void bkt_init_search_trees(const qctx_t* c, ws_t* ws)
{
    if (g_bfs == 0 || c->idx->tree_kind != ORA_BKT) {
        bkt_init_search_trees_default(c, ws);
        return;
    }
    const ora_bkt_node* nodes = (const ora_bkt_node*)c->idx->nodes;
    for (int i = 0; i < c->idx->tree_num; i++) {
        const int32_t start = c->idx->tree_starts[i];
        const ora_bkt_node* node = &nodes[start];
        ws->ntree++;
        if (node->childStart < 0) {
            pair_t p = {start, qdist(c, ws, node->centerid)};
            heap_insert(&ws->spt, p);
        } else {
            bkt_init_search_trees_bfs(c, ws, node);
        }
    }
}
